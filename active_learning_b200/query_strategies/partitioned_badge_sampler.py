from .coreset import PartitionedBADGEQuery
from .strategy import Strategy


class PartitionedBADGESampler(PartitionedBADGEQuery, Strategy):
    """Drop-in for active_learning/src/query_strategies/partitioned_badge_sampler.py (K2p + K3 + K5)."""
