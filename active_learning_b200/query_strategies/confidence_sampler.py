from .strategy import Strategy
from .uncertainty import ConfidenceQuery


class ConfidenceSampler(ConfidenceQuery, Strategy):
    """Drop-in for active_learning/src/query_strategies/confidence_sampler.py minus its line-41 bug
    (K1 least-confidence + K1b)."""
