from .maxherding import MaxHerdingQuery
from .strategy import Strategy


class MaxHerdingSampler(MaxHerdingQuery, Strategy):
    """MaxHerding (Bae, Noh & Sutherland, ECCV 2024) over CoreSet's pool (K22, K23); the sampler kwarg `sigma` is
    required."""
