from .coreset import BADGEQuery
from .strategy import Strategy


class BADGESampler(BADGEQuery, Strategy):
    """Drop-in for active_learning/src/query_strategies/badge_sampler.py (K2 + K3 + K5, factored)."""
