from .mase import MASEQuery
from .strategy import Strategy


class MASESampler(MASEQuery, Strategy):
    """Drop-in for active_learning/src/query_strategies/mase_sampler.py (K6 + K1b)."""
