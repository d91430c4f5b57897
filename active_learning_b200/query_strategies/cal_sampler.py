from .cal import CALQuery
from .strategy import Strategy


class CALSampler(CALQuery, Strategy):
    """CAL (Margatina et al., EMNLP 2021) over CoreSet's pool (K18, K19, K1b)."""
