from .coreset import PartitionedCoresetQuery
from .strategy import Strategy


class PartitionedCoresetSampler(PartitionedCoresetQuery, Strategy):
    """Drop-in for active_learning/src/query_strategies/partitioned_coreset_sampler.py."""
