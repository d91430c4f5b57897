from .mase import BASEQuery
from .strategy import Strategy


class BASESampler(BASEQuery, Strategy):
    """Drop-in for active_learning/src/query_strategies/base_sampler.py (K6 + per-class K1b)."""
