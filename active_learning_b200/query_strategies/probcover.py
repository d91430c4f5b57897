"""ProbCover (Yehuda et al., "Active Learning Through a Covering Lens", NeurIPS 2022) on the device (kernels K13, K14).

The pool's embeddings are L2-normalised and joined into the delta-ball graph, an edge (i, j) iff the euclidean distance of
the normalised rows is < delta (K13).  The greedy then repeatedly takes the row whose ball holds the most rows not yet
covered by a labeled or picked row's ball (the lowest position on ties) and covers them (K14).  Once every row is covered
the authors' `argmax` of an all-zero degree vector keeps returning position 0, a duplicate; here the greedy stops and
PoolQuery's random fill takes the rest of the budget.

Under --freeze_feature with no subsets the embeddings are round-invariant, so the graph stays on the device across rounds,
keyed on the pool and delta (CoreSet caches its N x N matrix under the same condition), and only K14 reruns.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from .coreset import PoolQuery


def probcover_delta(delta):
    """The sampler kwarg `delta` as a float: required, finite and > 0."""
    if delta is None:
        raise ValueError("ProbCoverSampler needs the sampler kwarg delta (the ball radius, finite and > 0)")
    delta = float(delta)
    if not (math.isfinite(delta) and delta > 0):
        raise ValueError(f"ProbCoverSampler: delta must be finite and > 0, got {delta}")
    return delta


class ProbCoverQuery(PoolQuery):
    """Greedy maximum coverage of the delta-ball graph over CoreSet's pool."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.delta = probcover_delta(kwargs.get("delta"))
        self._pc_cache = None

    def _graph(self, union):
        """(row_ptr, cols) of the pool's delta-ball graph, from the cache when the pool and delta are the cached ones."""
        cacheable = self.freeze_feature and self.subset_labeled is None and self.subset_unlabeled is None
        cache = getattr(self, "_pc_cache", None)
        if cacheable and cache is not None and cache[1] == self.delta and np.array_equal(cache[0], union):
            return cache[2], cache[3]
        self._pc_cache = None
        feats, _ = self._features(union.tolist())
        row_ptr, cols, _ = self.get_engine().probcover_graph(feats, self.delta)
        if cacheable:
            self._pc_cache = (union.copy(), self.delta, row_ptr, cols)
        return row_ptr, cols

    def _positions(self, union, is_lab, avail, budget):
        row_ptr, cols = self._graph(union)
        lab = torch.from_numpy(is_lab.astype(np.uint8)).to(row_ptr.device)
        picks, _steps = self.get_engine().probcover_select(row_ptr, cols, lab, budget)
        return picks
