"""`--strategy` dispatch, same contract as active_learning/src/query_strategies/get_strategy.py:
`get_strategy(name)` returns the class called `name`.  The twelve accelerated samplers (the seven of the
north-star path plus MASE / BASE / Balancing, SURVEY.md section 8f, MarginClustering and VAAL) and the default RandomSampler
are implemented; the reference's remaining class name resolves to a stub that raises a clear error (SURVEY.md section 8:
out of scope for this path)."""
from .badge_sampler import BADGESampler  # noqa: F401
from .balancing_sampler import BalancingSampler  # noqa: F401
from .base_sampler import BASESampler  # noqa: F401
from .confidence_sampler import ConfidenceSampler  # noqa: F401
from .coreset_sampler import CoresetSampler  # noqa: F401
from .entropy_sampler import EntropySampler  # noqa: F401
from .margin_clustering_sampler import MarginClusteringSampler  # noqa: F401
from .margin_sampler import MarginSampler  # noqa: F401
from .mase_sampler import MASESampler  # noqa: F401
from .partitioned_badge_sampler import PartitionedBADGESampler  # noqa: F401
from .partitioned_coreset_sampler import PartitionedCoresetSampler  # noqa: F401
from .random_sampler import RandomSampler  # noqa: F401
from .vaal_sampler import VAALSampler  # noqa: F401

ACCELERATED = ("MarginSampler", "ConfidenceSampler", "EntropySampler", "CoresetSampler",
               "PartitionedCoresetSampler", "BADGESampler", "PartitionedBADGESampler", "MASESampler", "BASESampler",
               "BalancingSampler", "MarginClusteringSampler", "VAALSampler")
NOT_ON_THIS_PATH = ("BalancedRandomSampler",)


def _out_of_scope(name):
    class _Stub:
        def __init__(self, *a, **k):
            raise NotImplementedError(
                f"{name} is not part of the accelerated query path; use the reference's own class")
    _Stub.__name__ = name
    return _Stub


def get_strategy(name):
    if name in NOT_ON_THIS_PATH:
        return _out_of_scope(name)
    cls = globals().get(name)
    if not isinstance(cls, type):
        raise NameError(f"name '{name}' is not defined")   # what the reference's eval(name) raises
    return cls
