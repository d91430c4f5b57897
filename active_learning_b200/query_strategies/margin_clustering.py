"""Margin clustering acquisition on the device (kernels K1, K7, K8): margin_clustering_sampler.py:47-90 of
active_learning/src/query_strategies (https://arxiv.org/abs/2107.14263).

The reference clusters the pool embeddings with sklearn's AgglomerativeClustering(n_clusters=20) -- Ward linkage over
the full tree: scipy's single-threaded pdist (a 25.6 GB condensed matrix at 80 000 rows) and nn_chain on the host --
then picks round-robin over the clusters, smallest cluster first, the smallest-margin row left in each.  Here one
pool forward yields logits and embeddings, K1 scores the margins, K7 builds the fp64 distances in HBM and K8 walks the
nearest-neighbour chain in one launch; the merge tree is scipy's bit for bit, so the labels are sklearn's
(include/alq.h).  The distances are the n x n matrix (8 n^2 bytes) when it fits the free device memory and scipy's
condensed vector (4 n (n - 1) bytes) otherwise, so on an 80 GB card the limit is about 140 000 rows (computed from the
card's memory, not measured), enough for ImageNet-LT's whole train set with subset_unlabeled unset; beyond it the query
raises AlqError.  The round robin is O(n log n) host NumPy over n margins.

In a ShardGroup of G > 1 ranks (with an engine that has the band kernel, `pdist_rows`) each rank forwards and scores its
row_range of the HAC rows, one all_gather_rows replicates the margins (and, in a round that clusters, the embeddings),
and ShardGroup.ward_labels splits K7 by pair-balanced bands of rows, sends the bands to rank 0 for K8 and broadcasts the
labels; every rank then runs the same round robin and returns the one-GPU picks.  When rank 0 cannot hold the distances
and the engine has the band calls (`band_alloc`, `nn_chain_banded`), each band stays on its rank and rank 0's K8 reads
the peers' bands through CUDA IPC peer memory, so the row limit becomes the ranks' memory together.
"""
from __future__ import annotations

import numpy as np

from .._lib import MODE_MARGIN, AlqError
from .strategy import EngineMixin

N_CLUSTERS = 20     # margin_clustering_sampler.py:59


def round_robin(assignment: np.ndarray, margins: np.ndarray, budget: int):
    """The pick loop of margin_clustering_sampler.py:64-89: clusters visited by (size, id); pass k takes the k-th row of
    every cluster larger than k, rows of a cluster ordered by (margin, position); stop after `budget` picks.
    Returns (positions in pick order, the assignment of the rows not picked, in pool order)."""
    assignment = np.asarray(assignment)
    margins = np.asarray(margins, dtype=np.float32)
    if assignment.shape[0] != margins.shape[0]:
        raise ValueError(f"cluster assignment has {assignment.shape[0]} rows, the pool has {margins.shape[0]}")
    n = assignment.shape[0]
    budget = int(min(n, budget))
    if budget <= 0:
        return np.empty(0, dtype=np.int64), assignment.copy()
    ids, inv, counts = np.unique(assignment, return_inverse=True, return_counts=True)
    visit = np.lexsort((ids, counts))                   # cluster visiting order: (count, id)
    visit_rank = np.empty(len(ids), dtype=np.int64)
    visit_rank[visit] = np.arange(len(ids))
    # rank of each row inside its cluster by (margin, position): order rows by (cluster, margin, position)
    by = np.lexsort((np.arange(n), margins, inv))
    first = np.zeros(len(ids), dtype=np.int64)
    first[1:] = np.cumsum(counts)[:-1]
    rank_in = np.empty(n, dtype=np.int64)
    rank_in[by] = np.arange(n) - first[inv[by]]
    key = rank_in * len(ids) + visit_rank[inv]
    picks = np.argsort(key, kind="stable")[:budget]
    keep = np.ones(n, dtype=bool)
    keep[picks] = False
    return picks.astype(np.int64), assignment[keep]


class MarginClusteringQuery(EngineMixin):
    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.saved_pairwise_l2_dist = None
        self.freeze_feature = kwargs["freeze_feature"]
        self.subset_labeled = kwargs["subset_labeled"]
        self.subset_unlabeled = kwargs["subset_unlabeled"]
        self.cluster_assignment = None

    # ---- margin_clustering_sampler.py:47-90 --------------------------------------------------------------
    def _hac_rows(self):
        if self.subset_unlabeled is None:
            return self.available_query_idxs(boolean=False, shuffle=False)
        return sorted(self.available_query_idxs(boolean=False, shuffle=True)[:self.subset_unlabeled])

    def query(self, budget):
        group = getattr(self, "_shard_group", None)
        if group is not None and group.world_size > 1:
            if not hasattr(self.get_engine(), "pdist_rows"):
                raise AlqError("MarginClusteringSampler runs on one GPU with this engine: it has no band kernel "
                               "(pdist_rows) to split Ward clustering's distances over a group; query it from a single "
                               "rank")
            return self._query_sharded(budget, group)
        idxs_for_hac = self._hac_rows()
        eng = self.get_engine()
        self.feature_net.eval()
        logits, emb = self._forward_pool(idxs_for_hac, self.feature_net, want_features=True)
        margins = eng.score_softmax(logits, MODE_MARGIN).cpu().numpy()
        if self.cluster_assignment is None or self.subset_unlabeled:
            # cluster in the first round, or every round when a random subset is drawn (:56-59)
            cluster_assignment = eng.ward_labels(emb, N_CLUSTERS)
        else:
            cluster_assignment = self.cluster_assignment
        budget = int(min(len(idxs_for_hac), budget))
        picks, self.cluster_assignment = round_robin(cluster_assignment, margins, budget)
        query_idxs = list(np.asarray(idxs_for_hac, dtype=np.int64)[picks])
        return query_idxs, budget

    # -- row-sharded variant: each rank forwards and scores n/G rows, K7 by bands, K8 on rank 0 ---------------
    def _query_sharded(self, budget, group):
        from ..sharding import digest
        idxs_for_hac = self._hac_rows()            # the same NumPy draws on every rank; ward_labels checks the digest
        n = len(idxs_for_hac)
        lo, hi = group.row_range(n)
        counts = [b - a for a, b in (group.row_range(n, r) for r in range(group.world_size))]
        clusters = self.cluster_assignment is None or bool(self.subset_unlabeled)
        eng = self.get_engine()
        self.feature_net.eval()
        logits, emb = self._forward_pool(idxs_for_hac[lo:hi], self.feature_net, want_features=True)
        margins = group.all_gather_rows(eng.score_softmax(logits, MODE_MARGIN), counts).cpu().numpy()
        if clusters:
            x = group.all_gather_rows(emb, counts)
            cluster_assignment = group.ward_labels(x, N_CLUSTERS, eng,
                                                   rows_digest=digest(np.asarray(idxs_for_hac, dtype=np.int64)))
        else:
            cluster_assignment = self.cluster_assignment
        budget = int(min(n, budget))
        picks, self.cluster_assignment = round_robin(cluster_assignment, margins, budget)
        return list(np.asarray(idxs_for_hac, dtype=np.int64)[picks]), budget
