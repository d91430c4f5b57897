from .bait import BAITQuery
from .strategy import Strategy


class BAITSampler(BAITQuery, Strategy):
    """BAIT (Ash, Goel, Krishnamurthy & Kakade, NeurIPS 2021) over CoreSet's pool (K24, K25, K26); the sampler kwarg
    `lamb` defaults to 1.0."""
