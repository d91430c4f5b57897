from .coreset import CoresetQuery
from .strategy import Strategy


class CoresetSampler(CoresetQuery, Strategy):
    """Drop-in for active_learning/src/query_strategies/coreset_sampler.py (K3 + K4)."""
