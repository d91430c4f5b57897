"""TypiClust (Hacohen, Dekel & Weinshall, "Active Learning on a Budget: Opposite Strategies Suit High and Low Budgets",
ICML 2022) on the device (kernels K5, K15, K16, K17).

The pool is CoreSet's (`get_idxs_for_coreset`: the same two shuffles, subset_labeled / subset_unlabeled honoured).  Its
embeddings are L2-normalised as ProbCover normalises them and clustered by k-means into K = min(|labeled| + budget,
MAX_NUM_CLUSTERS) clusters: k-means++ seeding is CoresetQuery's D^2 cold start (one np.random.choice(n), then K - 1
np.random.random_sample uniforms), then Lloyd's loop with exact fp64 assignments (K15) and sequential fp64 means (K16)
until no label changes, at most MAX_ITER assignments.

Selection follows the authors' loop: clusters with more than MIN_CLUSTER_SIZE rows, ordered by (labeled rows ascending,
size descending, id ascending), are visited cyclically; each visit takes the cluster's most typical available, unpicked
row, typicality = 1 / (mean squared distance to its k = min(K_NN, m // 2) nearest such rows + 1e-5) (K17, one launch per
cycle of the walk).  Two deliberate deviations, both where the authors' loop would index an empty cluster and fail: a
visit to a cluster with no row left is skipped and uses no budget, and once every kept cluster is exhausted the rest of
the budget is `np.random.choice(available-and-unpicked positions ascending, rest, replace=False)`, ProbCover's fill.

K changes with the labeled set and the seeding draws every round, so nothing but the embedding cache is kept across
rounds.  In a ShardGroup every rank runs the whole query on its own GPU and returns the same picks.
"""
from __future__ import annotations

import numpy as np
import torch

from .coreset import CoresetQuery


def cluster_order(labels, is_lab, k, min_size):
    """The kept cluster ids in visiting order: size > min_size, then (labeled rows ascending, size descending, id)."""
    size = np.bincount(labels, minlength=k)
    existing = np.bincount(labels[is_lab], minlength=k)
    ids = np.flatnonzero(size > min_size)
    return ids[np.lexsort((ids, -size[ids], existing[ids]))]


class TypiClustQuery(CoresetQuery):
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

    def query(self, budget):
        union = np.asarray(self.get_idxs_for_coreset(), dtype=np.int64)      # RNG: two permutations
        is_lab = self.already_labeled_idxs(boolean=True)[union]
        avail = self.available_query_idxs(boolean=True)[union]
        budget = int(min(int(avail.sum()), budget))
        if budget <= 0:
            return [], 0
        eng = self.get_engine()
        feats, _ = self._features(union.tolist())
        xhat = eng.normalize(feats)
        n = len(union)
        k = min(int(is_lab.sum()) + budget, self.MAX_NUM_CLUSTERS)
        first = int(np.random.choice(n))                                      # CoresetQuery's D^2 cold start
        unif = np.random.random_sample(k - 1)
        labels, _, _, _ = eng.kmeans(xhat, first, unif, k, self.MAX_ITER)
        labels = labels.cpu().numpy().astype(np.int64)
        picks = self._walk(xhat, labels, is_lab, avail, budget)
        rest = budget - len(picks)
        if rest > 0:                     # every kept cluster exhausted: the deliberate deviation above
            free = avail.copy()
            free[picks] = False
            picks = np.concatenate([picks, np.random.choice(np.flatnonzero(free), rest, replace=False)])
        labeled_idxs_cur_rd = union[picks].tolist()
        return labeled_idxs_cur_rd, len(labeled_idxs_cur_rd)
