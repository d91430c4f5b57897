"""NumPy statement of TypiClustSampler's query (active_learning_b200/query_strategies/typiclust.py, kernels K5, K15, K16,
K17), written from Hacohen, Dekel & Weinshall, "Active Learning on a Budget" (ICML 2022) and the authors' selection loop.
Matching sklearn's k-means or faiss's fp32 distances is not a goal (DESIGN section 2).

  pool       CoreSet's union (two shuffles), the budget clamped to the available rows, xhat = probcover_oracle.normalize;
  clusters   K = min(|labeled| + budget, MAX_NUM_CLUSTERS);
             seeding: CoresetQuery's D^2 cold start (np.random.choice(n), then K - 1 np.random.random_sample), the picks
             in pick order are the centres (`seed`);
             assignment: label_i = argmin_c exact_d2(xhat_i, c) (K7's pair arithmetic), ties to the lowest centre;
             update: centre_c = fl32(S_c / m_c), S_c = np.cumsum of the member rows in ascending row order in fp64, an
             empty cluster keeps its centre;
             Lloyd: assign, then update and assign while a label changed, at most MAX_ITER assignments;
  selection  the clusters with size > MIN_CLUSTER_SIZE ordered by (labeled rows ascending, size descending, id ascending),
             visited cyclically; a visit takes argmax typicality among the cluster's available, unpicked rows (lowest
             position on ties): typicality = 1 / (mean + 1e-5), mean = the ascending fp64 sum of the k = min(K_NN, m // 2)
             smallest exact squared distances to the other such rows / k; m = 1 takes the row (typicality 0);
  deviations a visit to an exhausted cluster is skipped without using budget; once every kept cluster is exhausted the
             rest is np.random.choice(available-and-unpicked positions ascending, rest, replace=False).

`authors_select` restates the authors' loop literally (np.unique, np.bincount, a lexsort for pandas' sort, brute-force
fp64 k-NN for faiss); while no kept cluster runs dry it equals `select`.  `assign_decide` is K15's band decision and
`exact_argmin` the assignment by brute force (`exact_d2_table`), for rows and centres of any norm.
"""
import numpy as np
import torch

import probcover_oracle as P
from oracle import al_oracle as O

MAX_NUM_CLUSTERS = 500
MIN_CLUSTER_SIZE = 5
K_NN = 20
MAX_ITER = 100

normalize = P.normalize
exact_d2 = P.exact_d2


# ---- clusters --------------------------------------------------------------------------------------------------------
def seed(xhat, first, uniforms, k):
    """k-means++ seeding: centre 0 is row `first`, then one D^2 draw per uniform (k - 1), exactly as CoresetQuery's cold
    start (al_oracle.coreset_streaming).  Rows, in pick order."""
    lab = np.zeros(xhat.shape[0], dtype=bool)
    lab[int(first)] = True
    rest = O.coreset_streaming(torch.from_numpy(np.ascontiguousarray(xhat)), lab, k - 1, randomize=True,
                               uniforms=np.asarray(uniforms, dtype=np.float64))
    return np.asarray([int(first)] + rest, dtype=np.int64)


def _screen_d2(x, c):
    x64, c64 = x.astype(np.float64), c.astype(np.float64)
    return (x64 * x64).sum(1)[:, None] + (c64 * c64).sum(1)[None, :] - 2.0 * (x64 @ c64.T)


def nearest_exact(x, c, want=1):
    """Per row of x, the `want` smallest exact_d2 values to the rows of c (ascending) and, for want == 1, the lowest
    column of the minimum.  An fp64 GEMM screens the pairs (its error is far below 1e-9 for rows of norm <= 1); only the
    columns within 1e-9 of the row's want-th smallest screened value are recomputed exactly."""
    vals, arg = [], []
    for lo in range(0, x.shape[0], 512):
        xs = x[lo:lo + 512]
        d2 = _screen_d2(xs, c)
        kth = np.partition(d2, want - 1, axis=1)[:, want - 1] if want <= d2.shape[1] else np.full(len(xs), np.inf)
        ri, cj = np.nonzero(d2 <= kth[:, None] + 1e-9)
        ex = exact_d2(xs[ri], c[cj])
        for r in range(len(xs)):
            sel = ri == r
            e, j = ex[sel], cj[sel]
            o = np.lexsort((j, e))
            vals.append(e[o][:want])
            arg.append(int(j[o][0]))
    return vals, np.asarray(arg, dtype=np.int64)


def assign(xhat, centres):
    """label_i = the lowest c of the minimum exact fp64 d2(xhat_i, centre_c)."""
    return nearest_exact(xhat, centres)[1]


def update(xhat, labels, centres):
    """fl32(fp64 sequential sum of the members in ascending row order / m); an empty cluster keeps its centre."""
    out = centres.copy()
    for c in range(centres.shape[0]):
        rows = np.flatnonzero(labels == c)
        if len(rows):
            s = np.cumsum(xhat[rows].astype(np.float64), axis=0)[-1]
            out[c] = (s / len(rows)).astype(np.float32)
    return out


def lloyd(xhat, centres, max_iter=MAX_ITER):
    """(labels, centres, assignments) of Lloyd's loop from the given centres."""
    labels = np.full(xhat.shape[0], -1, dtype=np.int64)
    it = 0
    while True:
        new = assign(xhat, centres)
        it += 1
        changed = int((new != labels).sum())
        labels = new
        if changed == 0 or it >= max_iter:
            return labels, centres, it
        centres = update(xhat, labels, centres)


def kmeans(xhat, first, uniforms, k, max_iter=MAX_ITER):
    seeds = seed(xhat, first, uniforms, k)
    return lloyd(xhat, xhat[seeds].copy(), max_iter)


# ---- selection ---------------------------------------------------------------------------------------------------------
def typicality(xhat, rows, k_nn=K_NN):
    """Typicality of each of `rows` among `rows` (the argmax's candidates): 1 / (mean + 1e-5), mean = the ascending fp64
    sum of the k = min(k_nn, m // 2) smallest exact squared distances to the other rows (by position) / k."""
    rows = np.asarray(rows, dtype=np.int64)
    m = len(rows)
    if m == 1:
        return np.zeros(1)
    k = min(k_nn, m // 2)
    x = xhat[rows]
    vals, _ = nearest_exact(x, x, want=k + 1)       # the row itself is among its k + 1 nearest with d2 = 0
    out = np.empty(m)
    for i, v in enumerate(vals):
        v = list(v)
        v.remove(0.0)                                # drop one zero: the row itself (a duplicate keeps its own zero)
        s = 0.0
        for t in sorted(v)[:k]:
            s += t
        out[i] = 1.0 / (s / k + 1e-5)
    return out


def cluster_order(labels, is_lab, k):
    size = np.bincount(labels, minlength=k)
    existing = np.bincount(labels[is_lab], minlength=k)
    ids = np.flatnonzero(size > MIN_CLUSTER_SIZE)
    return ids[np.lexsort((ids, -size[ids], existing[ids]))]


def select(xhat, labels, k, is_lab, avail, budget, typ=typicality):
    """The cyclic walk, one typicality per visit; positions in pick order (fewer than budget once every kept cluster is
    exhausted)."""
    order = cluster_order(labels, is_lab, k)
    free = np.asarray(avail, dtype=bool).copy()
    picks = []
    while len(picks) < budget:
        took = False
        for c in order:
            if len(picks) == budget:
                break
            cand = np.flatnonzero(free & (labels == c))
            if not len(cand):
                continue                                 # deviation: an exhausted cluster uses no budget
            p = int(cand[int(np.argmax(typ(xhat, cand)))])
            picks.append(p)
            free[p] = False
            took = True
        if not took:
            break
    return np.asarray(picks, dtype=np.int64)


def authors_select(features, clusters, lset_size, budget, k_nn=K_NN):
    """The authors' TypiClust selection loop restated without pandas: the labeled rows are positions [0, lset_size) of
    `features`, the unlabeled ones follow.  faiss's k-NN is brute-force exact fp64 d2 (k + 1 nearest, the first dropped)
    and the row mean is the ascending sum / k."""
    labels = np.copy(clusters)
    existing_indices = np.arange(lset_size)
    cluster_ids, cluster_sizes = np.unique(labels, return_counts=True)
    cluster_labeled_counts = np.bincount(labels[existing_indices], minlength=int(cluster_ids.max()) + 1)[cluster_ids]
    keep = cluster_sizes > MIN_CLUSTER_SIZE
    ids, sizes, existing = cluster_ids[keep], cluster_sizes[keep], cluster_labeled_counts[keep]
    order = np.lexsort((-sizes, existing))                 # sort_values(['existing_count', 'neg_cluster_size']), stable
    ids = ids[order]
    labels[existing_indices] = -1
    selected = []
    for i in range(budget):
        cluster = ids[i % len(ids)]
        indices = (labels == cluster).nonzero()[0]
        rel = features[indices]
        kk = min(k_nn, len(indices) // 2)
        if kk == 0:
            idx = indices[0]
        else:
            d2 = np.stack([exact_d2(np.repeat(rel[r:r + 1], len(rel), axis=0), rel) for r in range(len(rel))])
            knn = np.sort(d2, axis=1)[:, 1:kk + 1]
            mean = np.cumsum(knn, axis=1)[:, -1] / kk
            idx = indices[np.argmax(1 / (mean + 1e-5))]
        selected.append(idx)
        labels[idx] = -1
    return np.asarray(selected, dtype=np.int64)


def query_positions(emb, is_lab, avail, budget, seed_rows=None):
    """Positions in the pool that the query returns, in order, drawing from NumPy's global RNG as the sampler does.
    `seed_rows(xhat, first, uniforms, k)` replaces `seed` where a test supplies the seeding's rows."""
    budget = int(min(int(np.sum(avail)), budget))
    if budget <= 0:
        return np.zeros(0, dtype=np.int64)
    xhat = normalize(emb)
    n = xhat.shape[0]
    k = min(int(np.sum(is_lab)) + budget, MAX_NUM_CLUSTERS)
    first = int(np.random.choice(n))
    unif = np.random.random_sample(k - 1)
    rows = (seed_rows or seed)(xhat, first, unif, k)
    labels, _, _ = lloyd(xhat, xhat[rows].copy())
    picks = select(xhat, labels, k, np.asarray(is_lab, dtype=bool), avail, budget)
    return P.random_fill(picks, avail, budget)


# ---- K15's band ----------------------------------------------------------------------------------------------------------
def assign_decide(d, nrm_rows, cn, g):
    """K15's epilogue for the fp32 dot products g [n, K] of rows with nrm2 `nrm_rows` [n] and centres with cn [K] at
    padded width d, in fp64: (decided, c1) -- a row is decided when its second smallest lower bound exceeds its smallest
    upper bound, and then its label is c1."""
    coef = 2.0 * P.screen_bound(d, 1.0, 1.0) * (1.0 + 1e-6)
    ni, nc = np.asarray(nrm_rows, dtype=np.float64)[:, None], np.asarray(cn, dtype=np.float64)[None, :]
    d2 = (ni + nc) - 2.0 * np.asarray(g, dtype=np.float32).astype(np.float64)
    b = coef * (np.sqrt(ni) * np.sqrt(nc)) + 1e-9
    up, low = d2 + b, d2 - b
    u = up.min(axis=1)
    srt = np.sort(low, axis=1)
    l2 = srt[:, 1] if low.shape[1] > 1 else np.full(low.shape[0], np.inf)
    c1 = np.argmin(low, axis=1)
    return l2 > u, c1


def exact_d2_table(x, c, chunk=256):
    """[n, K] exact_d2(x_i, c_c) for every pair, by brute force (no screen, so any norm): per chunk of rows the sums
    d = a - b, s = s + d * d, k ascending, in fp64."""
    x, c = np.asarray(x, dtype=np.float32), np.asarray(c, dtype=np.float32)
    c64 = c.astype(np.float64)
    out = np.empty((x.shape[0], c.shape[0]))
    for lo in range(0, x.shape[0], chunk):
        xs = x[lo:lo + chunk].astype(np.float64)
        s = np.zeros((xs.shape[0], c.shape[0]))
        for k in range(x.shape[1]):
            df = xs[:, k, None] - c64[None, :, k]
            s = s + df * df
        out[lo:lo + chunk] = s
    return out


def exact_argmin(x, c, chunk=256):
    """label_i = the lowest c of the minimum exact_d2(x_i, c_c) over ALL centres (exact_d2_table's brute force)."""
    return np.argmin(exact_d2_table(x, c, chunk), axis=1).astype(np.int64)     # the first minimum: the lowest centre
