"""Class-balanced random acquisition on the device (kernel K10): the query of balanced_random_sampler.py:17-101 of
active_learning/src/query_strategies.  The reference itself calls it a baseline that cheats: it reads the labels of
the whole pool.

The reference converts the labels to a float tensor, counts the available rows per class with np.unique, raises a
threshold one step at a time until the per-class budgets add up to the query budget, and then, for every class, scans
the whole pool with `torch.where(labels == c, avail, False).nonzero()` and keeps a random prefix of the rows it found.
Here the labels go to the device once, K10 counts the classes in one pass, the threshold is found in closed form, and
K10 gathers every class's rows in one more pass.  What has to stay on the host is kept literally: NumPy's argsort of
the counts (its order among tied counts decides which classes get one more row) and the `torch.randperm(n_c)` draws
from torch's default CPU generator, one per class with a non-zero budget, classes ascending.  So the picks and the torch
RNG state afterwards equal the reference's; NumPy's RNG is not touched.
"""
from __future__ import annotations

import numpy as np
import torch

from .._lib import AlqError
from .strategy import EngineMixin


def balanced_class_budgets(counts, budget, num_classes):
    """Per-class budgets of balanced_random_sampler.py:43-72 (int32 [num_classes]), without its loop.

    With S(t) = sum_c min(count_c, t), the reference's loop stops at the smallest t >= budget // num_classes with
    S(t + 1) >= budget and gives the `budget - S(t)` classes that come last in `np.argsort(counts)` t + 1 rows, every
    other class min(count_c, t).  The argsort is the reference's own call on the same float64 array with the default
    kind: among tied counts its order is NumPy's, whatever that is on this host."""
    counts = np.asarray(counts, dtype=np.float64).reshape(-1)
    c = int(num_classes)
    budget = int(budget)
    if counts.size != c:
        raise ValueError(f"need {c} class counts, got {counts.size}")
    total = int(counts.sum())
    if budget < 0 or budget > total:
        raise ValueError(f"budget {budget} outside [0, {total}] (the available rows)")
    sort_idxs = np.argsort(counts)
    sorted_counts = counts[sort_idxs]
    reverse_sort_idxs = np.empty_like(sort_idxs)
    reverse_sort_idxs[sort_idxs] = np.arange(c)

    def level(t):
        return int(np.minimum(sorted_counts, t).sum())

    lo = budget // c                       # S(lo) <= c * lo <= budget
    hi = max(lo, int(sorted_counts[-1]))   # S(hi + 1) = total >= budget
    while lo < hi:                         # smallest t in [lo, hi] with S(t + 1) >= budget
        mid = (lo + hi) // 2
        if level(mid + 1) >= budget:
            hi = mid
        else:
            lo = mid + 1
    thres = lo
    oneadd = budget - level(thres)
    per_class = np.where(sorted_counts <= thres, sorted_counts, thres)
    if oneadd > 0:
        per_class[-oneadd:] = thres + 1
    return per_class[reverse_sort_idxs].astype(np.int32)


def _host_labels(targets):
    """The dataset's targets as a host int64 array: one conversion of a list, none of an array or tensor."""
    if isinstance(targets, torch.Tensor):
        return targets.detach().cpu().reshape(-1).to(torch.int64).numpy()
    return np.asarray(targets).reshape(-1).astype(np.int64, copy=False)


class BalancedRandomQuery(EngineMixin):
    """balanced_random_sampler.py: the same number of random rows from every class (as near as the class sizes allow)."""

    def query(self, budget):
        avail_h = np.ascontiguousarray(self.available_query_idxs(boolean=True), dtype=bool)
        budget = int(min(int(avail_h.sum()), budget))
        if budget <= 0:
            self.logger.info(f"Number of queried images: {max(budget, 0)}")
            return [], 0
        c = int(self.num_classes)
        labels_h = _host_labels(self.al_set.targets)
        if labels_h.size != avail_h.size:
            raise ValueError(f"the pool has {avail_h.size} rows but its targets hold {labels_h.size} labels")
        eng = self.get_engine()
        dev = self._query_device()
        # out-of-range labels stay out of range in int32, so the device check sees them
        labels = torch.from_numpy(np.clip(labels_h, -1, c).astype(np.int32)).to(dev)
        avail = torch.from_numpy(avail_h.view(np.uint8)).to(dev)
        try:
            counts = eng.class_counts(labels, avail, c).cpu().numpy()
        except AlqError:
            bad = np.flatnonzero(avail_h & ((labels_h < 0) | (labels_h >= c)))
            if bad.size:
                raise IndexError(f"pool row {int(bad[0])} is available for the query but its label {int(labels_h[bad[0]])} "
                                 f"is outside [0, {c})") from None
            raise
        k = balanced_class_budgets(counts, budget, c)
        # the reference's draws, in its order: randperm(n_c) for every class with a non-zero budget, classes ascending
        perms = [torch.randperm(int(counts[cls]))[:int(k[cls])] for cls in np.flatnonzero(k > 0)]
        perm = torch.cat(perms) if perms else torch.empty(0, dtype=torch.int64)
        picks = eng.class_pick(labels, avail, k, perm).cpu().numpy()
        if picks.size != budget or (picks < 0).any():
            raise RuntimeError("class_pick returned rows outside the pool: the class counts changed between the calls")
        self.logger.info(f"Number of queried images: {budget}")
        return picks.astype(np.int64).tolist(), budget
