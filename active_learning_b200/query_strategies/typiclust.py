"""TypiClust (Hacohen, Dekel & Weinshall, "Active Learning on a Budget: Opposite Strategies Suit High and Low Budgets",
ICML 2022) on the device (kernels K5, K15, K16, K17).

The pool's embeddings are L2-normalised as ProbCover normalises them and clustered by k-means into K = min(|labeled| +
budget, MAX_NUM_CLUSTERS) clusters: PoolQuery's k-means++ seeding draws, then Lloyd's loop with exact fp64 assignments
(K15) and sequential fp64 means (K16) until no label changes, at most MAX_ITER assignments.

Selection follows the authors' loop: clusters with more than MIN_CLUSTER_SIZE rows, ordered by (labeled rows ascending,
size descending, id ascending), are visited cyclically; each visit takes the cluster's most typical available, unpicked
row, typicality = 1 / (mean squared distance to its k = min(K_NN, m // 2) nearest such rows + 1e-5) (K17, one launch per
cycle of the walk).  A visit to a cluster with no row left, where the authors' loop would index an empty cluster and fail,
is skipped and uses no budget; once every kept cluster is exhausted PoolQuery's random fill takes the rest of the budget.

K changes with the labeled set and the seeding draws every round, so nothing but the embedding cache is kept across
rounds.
"""
from __future__ import annotations

import numpy as np
import torch

from .coreset import PoolQuery


def cluster_order(labels, is_lab, k, min_size):
    """The kept cluster ids in visiting order: size > min_size, then (labeled rows ascending, size descending, id)."""
    size = np.bincount(labels, minlength=k)
    existing = np.bincount(labels[is_lab], minlength=k)
    ids = np.flatnonzero(size > min_size)
    return ids[np.lexsort((ids, -size[ids], existing[ids]))]


class TypiClustQuery(PoolQuery):
    """The most typical row of each uncovered k-means cluster of CoreSet's pool."""
    MAX_NUM_CLUSTERS = 500
    MIN_CLUSTER_SIZE = 5
    K_NN = 20
    MAX_ITER = 100

    def _walk(self, xhat, labels, is_lab, avail, budget):
        """The cyclic walk over the kept clusters; positions in pick order (possibly fewer than budget)."""
        eng = self.get_engine()
        order = cluster_order(labels, is_lab, int(labels.max()) + 1 if len(labels) else 0, self.MIN_CLUSTER_SIZE)
        free = avail.copy()
        picks = []
        while len(picks) < budget and len(order):
            pos = np.flatnonzero(free)
            pos = pos[np.argsort(labels[pos], kind="stable")]            # free rows grouped by cluster, ascending
            cut = np.searchsorted(labels[pos], np.arange(int(labels.max()) + 2))
            live = [c for c in order if cut[c + 1] > cut[c]][:budget - len(picks)]
            if not live:
                break
            rows = np.concatenate([pos[cut[c]:cut[c + 1]] for c in live])
            goff = np.zeros(len(live) + 1, dtype=np.int64)
            goff[1:] = np.cumsum([cut[c + 1] - cut[c] for c in live])
            _, best = eng.typicality(xhat, torch.as_tensor(rows.astype(np.int32), device=xhat.device), goff, self.K_NN)
            new = rows[best]
            picks += new.tolist()
            free[new] = False
        return np.asarray(picks, dtype=np.int64)

    def _positions(self, union, is_lab, avail, budget):
        feats, _ = self._features(union.tolist())
        xhat = self.get_engine().normalize(feats)
        k = min(int(is_lab.sum()) + budget, self.MAX_NUM_CLUSTERS)
        labels, _, _, _ = self._kmeans(xhat, k, self.MAX_ITER)
        labels = labels.cpu().numpy().astype(np.int64)
        return self._walk(xhat, labels, is_lab, avail, budget)
