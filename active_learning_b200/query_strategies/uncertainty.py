"""Softmax-uncertainty acquisition on the device (kernels K1 + K1b).

Query skeleton of active_learning/src/query_strategies/margin_sampler.py:19-45: pool indices in
loader order -> frozen-network forward -> per-row score -> the `budget` smallest scores, ascending,
ties by pool position -> global indices.  What differs from the reference is only *where* the
tail runs: logits stay in a device slab, the score and the top-B selection are CUDA kernels, and
B int32 positions are the only thing that returns to the host.
"""
from __future__ import annotations

import numpy as np
import torch

from .._lib import MODE_ENTROPY, MODE_LEAST_CONFIDENCE, MODE_MARGIN, AlqError  # noqa: F401
from .strategy import EngineMixin


class UncertaintyQuery(EngineMixin):
    MODE = MODE_MARGIN
    SHUFFLE_POOL = False       # margin_sampler.py:21 passes shuffle=False

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.cache_embeddings = kwargs.get("cache_embeddings", True)
        self.channels_last = kwargs.get("channels_last", True)

    def query(self, budget):
        idxs_for_query = self.available_query_idxs(boolean=False, shuffle=self.SHUFFLE_POOL)
        budget = int(min(len(idxs_for_query), budget))
        if budget <= 0:
            return [], 0
        group = getattr(self, "_shard_group", None)
        if group is not None and group.world_size > 1:
            pos = self._query_sharded(idxs_for_query, budget, group)
        else:
            self.net.eval()
            logits, _ = self._forward_pool(idxs_for_query, self.net, want_features=False)
            self.net.train()                               # margin_sampler.py:38
            eng = self.get_engine()
            pos = self._tail(eng, logits, budget)[1].cpu().numpy()
        labeled_idxs = np.asarray(idxs_for_query)[pos].tolist()
        return labeled_idxs, budget

    def _tail(self, eng, logits, b):
        """(scores, positions of the b smallest in stable order): K1 + K1b, one fused launch where the engine has it."""
        if hasattr(eng, "uncertainty_tail"):
            return eng.uncertainty_tail(logits, self.MODE, b)
        scores = eng.score_softmax(logits, self.MODE)
        return scores, eng.select_smallest(scores, b)

    # -- row-sharded variant: every rank scores N/G rows, one exchange for the global top-B ------
    def _query_sharded(self, idxs_for_query, budget, group):
        n = len(idxs_for_query)
        lo, hi = group.row_range(n)
        self.net.eval()
        logits, _ = self._forward_pool(idxs_for_query[lo:hi], self.net, want_features=False)
        self.net.train()
        eng = self.get_engine()
        if getattr(eng, "comm_ready", False) and hasattr(eng, "uncertainty_tail_sharded"):
            # K1 + K1b + the exchange as one launch per rank (peer-memory windows); one barrier first: the forward passes
            # of the ranks can drift apart by seconds and the in-kernel waits are bounded
            import torch.distributed as dist
            sizes = [b_ - a_ for a_, b_ in (group.row_range(n, q) for q in range(group.world_size))]
            dist.barrier(group=group.pg)
            try:
                _, gpos = eng.uncertainty_tail_sharded(logits, self.MODE, budget, lo, min(sizes), max(sizes))
                host = gpos.cpu().numpy()
                eng.comm_check()
                return host.astype(np.int64) & 0xFFFFFFFF
            except AlqError:                        # a peer never showed up, or a budget above 16 384 that does not
                pass                                # fuse (declined on every rank alike): the collective path below
        b_loc = min(budget, hi - lo)
        scores, pos_loc = self._tail(eng, logits, b_loc)
        return group.merge_smallest(scores, pos_loc, lo, budget, eng, rendezvous=True)


class MarginQuery(UncertaintyQuery):
    """margin_sampler.py: p(1) - p(2), smallest first."""
    MODE = MODE_MARGIN
    SHUFFLE_POOL = False


class ConfidenceQuery(UncertaintyQuery):
    """confidence_sampler.py with line 41 removed (SURVEY.md finding 2): p(1), smallest first.
    The pool order is the shuffled one (`available_query_idxs()` default, :19), so ties resolve by
    position in that permutation, exactly as a stable sort of the reference's vector would."""
    MODE = MODE_LEAST_CONFIDENCE
    SHUFFLE_POOL = True


class EntropyQuery(UncertaintyQuery):
    """NEW (absent from the reference, SURVEY.md finding 1 / section 8 row A3): largest softmax
    entropy first == ascending sum_c p_c log p_c; MarginSampler's skeleton otherwise."""
    MODE = MODE_ENTROPY
    SHUFFLE_POOL = False
