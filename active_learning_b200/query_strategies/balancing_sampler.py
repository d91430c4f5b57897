from .balancing import BalancingQuery
from .strategy import Strategy


class BalancingSampler(BalancingQuery, Strategy):
    """Drop-in for active_learning/src/query_strategies/balancing_sampler.py (K3 distance fields + masked ratio arg-min)."""
