from .strategy import Strategy
from .uncertainty import MarginQuery


class MarginSampler(MarginQuery, Strategy):
    """Drop-in for active_learning/src/query_strategies/margin_sampler.py (K1 margin + K1b)."""
