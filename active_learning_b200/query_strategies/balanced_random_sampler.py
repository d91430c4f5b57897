from .balanced_random import BalancedRandomQuery
from .strategy import Strategy


class BalancedRandomSampler(BalancedRandomQuery, Strategy):
    """Drop-in for active_learning/src/query_strategies/balanced_random_sampler.py (K10)."""
