"""`--strategy` dispatch, same contract as active_learning/src/query_strategies/get_strategy.py:
`get_strategy(name)` returns the class called `name`.  Every class name the reference dispatches is implemented: the
thirteen accelerated samplers (the seven of the north-star path plus MASE / BASE / Balancing, SURVEY.md section 8f,
MarginClustering, VAAL and BalancedRandom) and the default RandomSampler.  ProbCoverSampler, TypiClustSampler,
CALSampler and ALFAMixSampler are this project's additions (no reference counterpart; ProbCoverSampler needs the sampler
kwarg `delta`)."""
from .alfamix_sampler import ALFAMixSampler  # noqa: F401
from .badge_sampler import BADGESampler  # noqa: F401
from .balanced_random_sampler import BalancedRandomSampler  # noqa: F401
from .balancing_sampler import BalancingSampler  # noqa: F401
from .base_sampler import BASESampler  # noqa: F401
from .cal_sampler import CALSampler  # noqa: F401
from .confidence_sampler import ConfidenceSampler  # noqa: F401
from .coreset_sampler import CoresetSampler  # noqa: F401
from .entropy_sampler import EntropySampler  # noqa: F401
from .margin_clustering_sampler import MarginClusteringSampler  # noqa: F401
from .margin_sampler import MarginSampler  # noqa: F401
from .mase_sampler import MASESampler  # noqa: F401
from .partitioned_badge_sampler import PartitionedBADGESampler  # noqa: F401
from .partitioned_coreset_sampler import PartitionedCoresetSampler  # noqa: F401
from .probcover_sampler import ProbCoverSampler  # noqa: F401
from .random_sampler import RandomSampler  # noqa: F401
from .typiclust_sampler import TypiClustSampler  # noqa: F401
from .vaal_sampler import VAALSampler  # noqa: F401

ACCELERATED = ("MarginSampler", "ConfidenceSampler", "EntropySampler", "CoresetSampler",
               "PartitionedCoresetSampler", "BADGESampler", "PartitionedBADGESampler", "MASESampler", "BASESampler",
               "BalancingSampler", "MarginClusteringSampler", "VAALSampler", "BalancedRandomSampler",
               "ProbCoverSampler", "TypiClustSampler", "CALSampler", "ALFAMixSampler")
NOT_ON_THIS_PATH = ()


def get_strategy(name):
    cls = globals().get(name)
    if not isinstance(cls, type):
        raise NameError(f"name '{name}' is not defined")   # what the reference's eval(name) raises
    return cls
