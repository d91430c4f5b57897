"""Binding the accelerated query() implementations onto the REFERENCE's own Strategy base class.

The classes in ``active_learning_b200.query_strategies`` derive from a query-path-only Strategy.
A maintainer of the reference who wants to keep its training loop, checkpointing and Comet
logging and only swap the query tail does:

    import query_strategies.strategy as ref                       # the reference's module
    from active_learning_b200.integration import make_drop_in
    ACCEL = make_drop_in(ref.Strategy)
    # with VAAL as well:  make_drop_in(ref.Strategy, vaal_base=query_strategies.vaal_sampler.VAALSampler)
    # in query_strategies/get_strategy.py:   def get_strategy(name): return ACCEL.get(name) or eval(name)

See INTEGRATION.md.
"""
from __future__ import annotations

from .query_strategies.coreset import (BADGEQuery, CoresetQuery, PartitionedBADGEQuery,
                                       PartitionedCoresetQuery)
from .query_strategies.alfamix import ALFAMixQuery
from .query_strategies.balanced_random import BalancedRandomQuery
from .query_strategies.cal import CALQuery
from .query_strategies.balancing import BalancingQuery
from .query_strategies.margin_clustering import MarginClusteringQuery
from .query_strategies.mase import BASEQuery, MASEQuery
from .query_strategies.probcover import ProbCoverQuery
from .query_strategies.typiclust import TypiClustQuery
from .query_strategies.uncertainty import ConfidenceQuery, EntropyQuery, MarginQuery
from .query_strategies.vaal import VAALQuery

_MIXINS = {
    "MarginSampler": MarginQuery,
    "ConfidenceSampler": ConfidenceQuery,
    "EntropySampler": EntropyQuery,
    "CoresetSampler": CoresetQuery,
    "PartitionedCoresetSampler": PartitionedCoresetQuery,
    "BADGESampler": BADGEQuery,
    "PartitionedBADGESampler": PartitionedBADGEQuery,
    "MASESampler": MASEQuery,
    "BASESampler": BASEQuery,
    "BalancingSampler": BalancingQuery,
    "MarginClusteringSampler": MarginClusteringQuery,
    "BalancedRandomSampler": BalancedRandomQuery,
    "ProbCoverSampler": ProbCoverQuery,
    "TypiClustSampler": TypiClustQuery,
    "CALSampler": CALQuery,
    "ALFAMixSampler": ALFAMixQuery,
}


def make_drop_in(strategy_base, vaal_base=None):
    """{class name: class(mixin, strategy_base)} for every accelerated sampler.  With `vaal_base`, the reference's own
    VAALSampler class, the dict also holds "VAALSampler": class(VAALQuery, vaal_base): the reference's __init__ and
    parallel_train_fn build and train the VAE and the discriminator, and only query() is replaced."""
    out = {name: type(name, (mixin, strategy_base), {"__doc__": mixin.__doc__})
           for name, mixin in _MIXINS.items()}
    if vaal_base is not None:
        out["VAALSampler"] = type("VAALSampler", (VAALQuery, vaal_base), {"__doc__": VAALQuery.__doc__})
    return out
