"""ProbCover (Yehuda et al., "Active Learning Through a Covering Lens", NeurIPS 2022) on the device (kernels K13, K14).

The pool is CoreSet's (`get_idxs_for_coreset`: the same two shuffles, subset_labeled / subset_unlabeled honoured).  Its
embeddings are L2-normalised and joined into the delta-ball graph, an edge (i, j) iff the euclidean distance of the
normalised rows is < delta (K13).  The greedy then repeatedly takes the row whose ball holds the most rows not yet covered
by a labeled or picked row's ball (the lowest position on ties) and covers them (K14).

One deliberate deviation from the authors' loop: once every row is covered their `argmax` of an all-zero degree vector
keeps returning position 0, a duplicate.  Here the rest of the budget is drawn instead with
`np.random.choice(available-and-unpicked positions ascending, rest, replace=False)` -- the only NumPy draw after the pool's
two shuffles.

Under --freeze_feature with no subsets the embeddings are round-invariant, so the graph stays on the device across rounds,
keyed on the pool and delta (CoreSet caches its N x N matrix under the same condition), and only K14 reruns.  In a
ShardGroup every rank runs the whole query on its own GPU and returns the same picks.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from .coreset import CoresetQuery


def probcover_delta(delta):
    """The sampler kwarg `delta` as a float: required, finite and > 0."""
    if delta is None:
        raise ValueError("ProbCoverSampler needs the sampler kwarg delta (the ball radius, finite and > 0)")
    delta = float(delta)
    if not (math.isfinite(delta) and delta > 0):
        raise ValueError(f"ProbCoverSampler: delta must be finite and > 0, got {delta}")
    return delta


class ProbCoverQuery(CoresetQuery):
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

    def query(self, budget):
        union = np.asarray(self.get_idxs_for_coreset(), dtype=np.int64)      # RNG: two permutations
        is_lab = self.already_labeled_idxs(boolean=True)[union]
        avail = self.available_query_idxs(boolean=True)[union]
        budget = int(min(int(avail.sum()), budget))
        if budget <= 0:
            return [], 0
        row_ptr, cols = self._graph(union)
        lab = torch.from_numpy(is_lab.astype(np.uint8)).to(row_ptr.device)
        picks, _steps = self.get_engine().probcover_select(row_ptr, cols, lab, budget)
        rest = budget - len(picks)
        if rest > 0:                     # full coverage before the budget: the deliberate deviation above
            free = avail.copy()
            free[picks] = False
            picks = np.concatenate([picks, np.random.choice(np.flatnonzero(free), rest, replace=False)])
        labeled_idxs_cur_rd = union[picks].tolist()
        return labeled_idxs_cur_rd, len(labeled_idxs_cur_rd)
