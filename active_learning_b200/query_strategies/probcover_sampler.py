from .probcover import ProbCoverQuery
from .strategy import Strategy


class ProbCoverSampler(ProbCoverQuery, Strategy):
    """ProbCover (Yehuda et al., NeurIPS 2022) over CoreSet's pool (K13, K14); the sampler kwarg `delta` is required."""
