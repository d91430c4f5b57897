"""NumPy twin of the MarginClusteringSampler path (K7, K8, alq_ward_labels and the round robin), written from the
algorithms' definitions: scipy's pdist / nn_chain (Ward) / label, sklearn's _hc_cut, and the pick loop of
margin_clustering_sampler.py:64-89.  The CPU tier checks it against scipy and sklearn themselves and replays the
reference's goldens through it; the GPU tier checks the kernels against it bit for bit."""
import heapq

import numpy as np

N_CLUSTERS = 20


def pdist_square(x):
    """scipy's pdist(x, 'euclidean') as a full n x n fp64 matrix (diagonal 0): per pair, s summed k = 0, 1, ... as
    `d = a - b; s = s + d*d` (np.cumsum accumulates strictly left to right), then sqrt."""
    x = np.asarray(x, dtype=np.float64)
    n = x.shape[0]
    out = np.zeros((n, n), dtype=np.float64)
    for i in range(n - 1):
        diff = x[i] - x[i + 1:]
        s = np.cumsum(diff * diff, axis=1)[:, -1]
        out[i, i + 1:] = np.sqrt(s)
        out[i + 1:, i] = out[i, i + 1:]
    return out


def ward_nn_chain(dist):
    """scipy's nn_chain with the Ward update on a full square matrix (copied).  Returns (merge_xy [n-1, 2] int64 with
    x < y, merge_dist [n-1]) in the chain's discovery order, and the longest chain seen."""
    D = np.array(dist, dtype=np.float64, copy=True)
    n = D.shape[0]
    size = np.ones(n, dtype=np.int64)
    xy = np.empty((n - 1, 2), dtype=np.int64)
    md = np.empty(n - 1, dtype=np.float64)
    chain, longest = [], 0
    for k in range(n - 1):
        if not chain:
            chain.append(int(np.flatnonzero(size > 0)[0]))
        while True:
            x = chain[-1]
            if len(chain) > 1:
                y = chain[-2]
                cur = D[x, y]                        # ties go to the previous chain element
            else:
                y, cur = -1, np.inf
            row = np.where(size > 0, D[x], np.inf)
            row[x] = np.inf
            row[np.isnan(row)] = np.inf              # NaN never wins a strict '<'
            i = int(np.argmin(row))                  # lowest index among equal minima
            if row[i] < cur:
                cur, y = row[i], i
            if len(chain) > 1 and y == chain[-2]:
                break
            chain.append(y)
            longest = max(longest, len(chain))
        chain.pop()
        chain.pop()
        if x > y:
            x, y = y, x
        nx, ny = size[x], size[y]
        xy[k] = (x, y)
        md[k] = cur
        size[x] = 0
        size[y] = nx + ny
        live = np.flatnonzero(size > 0)
        live = live[live != y]
        ni = size[live]
        t = 1.0 / (nx + ny + ni)
        dx, dy = D[x, live], D[y, live]
        new = np.sqrt((ni + nx) * t * dx * dx + (ni + ny) * t * dy * dy - ni * t * cur * cur)
        D[y, live] = new
        D[live, y] = new
    return xy, md, longest


def linkage_from_merges(xy, md, n):
    """scipy's epilogue of nn_chain: stable sort by distance, then union-find relabelling -> Z [n-1, 4]."""
    order = np.argsort(md, kind="mergesort")
    parent = np.arange(2 * n - 1)
    sizes = np.ones(2 * n - 1, dtype=np.int64)
    nxt = n

    def find(v):
        while parent[v] != v:
            v = parent[v]
        return v

    Z = np.empty((n - 1, 4), dtype=np.float64)
    for r, k in enumerate(order):
        a, b = find(int(xy[k, 0])), find(int(xy[k, 1]))
        a, b = min(a, b), max(a, b)
        parent[a] = parent[b] = nxt
        sizes[nxt] = sizes[a] + sizes[b]
        Z[r] = (a, b, md[k], sizes[nxt])
        nxt += 1
    return Z


def hc_cut(n_clusters, children, n):
    """Cut of the full tree into n_clusters: repeatedly split the highest node (a heap of negated ids); cluster
    numbers follow the heap's final list order."""
    if n_clusters > n:
        raise ValueError(f"cannot extract {n_clusters} clusters from {n} leaves")
    children = np.asarray(children, dtype=np.int64)
    heap = [-(int(children[-1].max()) + 1)]
    for _ in range(n_clusters - 1):
        c0, c1 = children[-heap[0] - n]
        heapq.heappush(heap, -int(c0))
        heapq.heappushpop(heap, -int(c1))
    labels = np.zeros(n, dtype=np.int64)
    for lab, node in enumerate(heap):
        stack = [-node]
        while stack:
            v = stack.pop()
            if v < n:
                labels[v] = lab
            else:
                stack.extend(children[v - n].tolist())
    return labels


def ward_labels(x, n_clusters=N_CLUSTERS):
    """AgglomerativeClustering(n_clusters).fit(x).labels_ (Ward, full tree) through the twins above."""
    x = np.asarray(x, dtype=np.float32)
    n = x.shape[0]
    if n < max(2, n_clusters):
        raise ValueError(f"cannot extract {n_clusters} clusters from {n} rows")
    if not np.isfinite(x).all():
        raise ValueError("non-finite embeddings")
    xy, md, _ = ward_nn_chain(pdist_square(x))
    Z = linkage_from_merges(xy, md, n)
    return hc_cut(n_clusters, Z[:, :2].astype(np.int64), n)


def round_robin(assignment, margins, budget):
    """Pass by pass: clusters in (size, id) order, each still holding a row gives up its smallest-margin row (lowest
    position on ties); stop after `budget` picks.  Returns (positions, assignment of the rows left)."""
    assignment = np.array(assignment, copy=True)
    margins = np.asarray(margins, dtype=np.float32)
    budget = int(min(len(assignment), budget))
    ids, counts = np.unique(assignment, return_counts=True)
    visit = [ids[i] for i in sorted(range(len(ids)), key=lambda i: (counts[i], ids[i]))]
    queues = {}
    for c in visit:
        rows = np.flatnonzero(assignment == c)
        queues[c] = list(rows[np.argsort(margins[rows], kind="stable")])
    picks, k = [], 0
    while len(picks) < budget:
        for c in visit:
            if k < len(queues[c]) and len(picks) < budget:
                picks.append(int(queues[c][k]))
        k += 1
    left = np.ones(len(assignment), dtype=bool)
    left[picks] = False
    return np.asarray(picks, dtype=np.int64), assignment[left]


def shrinking_gap_line(n):
    """1-D points whose gaps shrink strictly, index 0 at the wide end: the nearest-neighbour chain started at 0 walks
    the whole line before its first merge (length n).  Integer coordinates (gaps n-1, n-2, ..., 1), exact in fp32."""
    gaps = np.arange(n - 1, 0, -1, dtype=np.int64)
    pos = np.concatenate([[0], np.cumsum(gaps)])
    return pos.astype(np.float32)[:, None]
