"""NumPy statement of ProbCoverSampler's query (active_learning_b200/query_strategies/probcover.py, kernels K13 / K14),
written from the algorithm of Yehuda et al., "Active Learning Through a Covering Lens" (NeurIPS 2022):

  normalise  lane l of 32 sums the fp64 squares of columns l, l + 32, .. in order, a butterfly (xor 16, 8, 4, 2, 1)
             adds the partials, norm = sqrt, xhat = fl32(x / norm) in fp64; a zero row stays zero;
  graph      an edge (i, j) iff scipy's fp64 euclidean distance of xhat_i, xhat_j is < delta (d = a - b, s = s + d * d,
             k ascending, then sqrt), as CSR with ascending columns;
  greedy     covered = the balls of the labeled rows; deg[x] = uncovered rows in N(x); each step stops if max deg = 0,
             else takes the lowest position c of the maximum and covers N(c);
  fill       the rest of the budget is np.random.choice(available-and-unpicked positions ascending, rest, replace=False).
"""
import numpy as np

LANES = 32


def normalize(x):
    x = np.asarray(x, dtype=np.float32)
    n, d = x.shape
    dp = -(-max(d, 1) // LANES) * LANES
    x64 = np.zeros((n, dp))
    x64[:, :d] = x
    sq = (x64 * x64).reshape(n, dp // LANES, LANES)
    s = np.zeros((n, LANES))
    for m in range(sq.shape[1]):
        s = s + sq[:, m, :]
    lanes = np.arange(LANES)
    for o in (16, 8, 4, 2, 1):
        s = s + s[:, lanes ^ o]
    norm = np.sqrt(s[:, 0])
    out = np.zeros((n, d), dtype=np.float32)
    nz = norm > 0
    out[nz] = (x[nz].astype(np.float64) / norm[nz, None]).astype(np.float32)
    return out


def exact_d2(a, b):
    """scipy's euclidean sum for row pairs (a[p], b[p]) of fp32 rows, in fp64, k ascending, no FMA."""
    a, b = np.asarray(a, dtype=np.float32), np.asarray(b, dtype=np.float32)
    s = np.zeros(a.shape[0])
    for k in range(a.shape[1]):
        df = a[:, k].astype(np.float64) - b[:, k].astype(np.float64)
        s = s + df * df
    return s


def ball_rows(xhat, delta, rows):
    """N(r) for each r in rows: the ascending columns j with dist(xhat_r, xhat_j) < delta.  A fp64 GEMM screens the pairs
    (its error is below 1e-12 for unit rows); pairs within 1e-9 of delta^2 are decided by exact_d2."""
    x64 = xhat.astype(np.float64)
    nrm = (x64 * x64).sum(axis=1)
    d2c = delta * delta
    out = []
    rows = np.asarray(rows, dtype=np.int64)
    for lo in range(0, len(rows), 1024):
        r = rows[lo:lo + 1024]
        d2 = nrm[r, None] + nrm[None, :] - 2.0 * (x64[r] @ x64.T)
        adj = d2 < d2c
        bi, bj = np.nonzero(np.abs(d2 - d2c) <= 1e-9 * d2c + 1e-9)
        if len(bi):
            adj[bi, bj] = np.sqrt(exact_d2(xhat[r[bi]], xhat[bj])) < delta
        out += [np.flatnonzero(a).astype(np.int32) for a in adj]
    return out


def graph(xhat, delta):
    """(row_ptr int64 [n + 1], cols int32 [nnz]) of the delta-ball graph of the normalised rows."""
    balls = ball_rows(xhat, delta, np.arange(xhat.shape[0]))
    row_ptr = np.zeros(len(balls) + 1, dtype=np.int64)
    row_ptr[1:] = np.cumsum([len(b) for b in balls])
    cols = np.concatenate(balls) if balls else np.zeros(0, dtype=np.int32)
    return row_ptr, cols.astype(np.int32)


def greedy(row_ptr, cols, labeled, budget):
    """The greedy coverage picks (positions, pick order); stops early when max deg = 0."""
    n = len(row_ptr) - 1
    rows_of = np.repeat(np.arange(n), np.diff(row_ptr))
    covered = np.zeros(n, dtype=bool)
    for r in np.flatnonzero(labeled):
        covered[cols[row_ptr[r]:row_ptr[r + 1]]] = True
    deg = np.bincount(rows_of, weights=~covered[cols], minlength=n).astype(np.int64)
    picks = []
    for _ in range(int(budget)):
        c = int(np.argmax(deg))
        if deg[c] == 0:
            break
        ys = cols[row_ptr[c]:row_ptr[c + 1]]
        ys = ys[~covered[ys]]
        covered[ys] = True
        nb = np.concatenate([cols[row_ptr[y]:row_ptr[y + 1]] for y in ys])
        deg -= np.bincount(nb, minlength=n)
        picks.append(c)
    return np.asarray(picks, dtype=np.int64)


def authors_greedy(edge_x, edge_y, n, labeled_pos, budget):
    """The authors' selection loop restated literally on an edge list (x -> y, both directions, self edges included),
    run while max deg > 0: np.isin / np.bincount / argmax, as in their ProbCover.select_samples."""
    edge_from_seen = np.isin(edge_x, labeled_pos)
    covered_samples = np.unique(edge_y[edge_from_seen])
    keep = ~np.isin(edge_y, covered_samples)
    cx, cy = edge_x[keep], edge_y[keep]
    selected = []
    for _ in range(int(budget)):
        degrees = np.bincount(cx, minlength=n)
        if degrees.max(initial=0) == 0:
            break
        cur = int(degrees.argmax())
        new_covered = cy[cx == cur]
        assert len(np.intersect1d(covered_samples, new_covered)) == 0
        keep = ~np.isin(cy, new_covered)
        cx, cy = cx[keep], cy[keep]
        covered_samples = np.concatenate([covered_samples, new_covered])
        selected.append(cur)
    return np.asarray(selected, dtype=np.int64)


def random_fill(picks, avail, budget):
    """The rest of the budget after full coverage: one np.random.choice over the available, unpicked positions."""
    picks = np.asarray(picks, dtype=np.int64)
    rest = int(budget) - len(picks)
    if rest <= 0:
        return picks
    free = np.asarray(avail, dtype=bool).copy()
    free[picks] = False
    return np.concatenate([picks, np.random.choice(np.flatnonzero(free), rest, replace=False)])


def query_positions(emb, is_lab, avail, budget, delta):
    """Positions in the pool that the query returns, in order (NumPy's global RNG drives only the fill)."""
    budget = int(min(int(np.sum(avail)), budget))
    if budget <= 0:
        return np.zeros(0, dtype=np.int64)
    row_ptr, cols = graph(normalize(emb), delta)
    return random_fill(greedy(row_ptr, cols, is_lab, budget), avail, budget)


# ---- the tensor-core screen's bound (K13) ----------------------------------------------------------------------------
def screen_bound(d, nrm_i, nrm_j):
    """|g - <xhat_i, xhat_j>| <= E for K13's 3xTF32 dot product g (DESIGN section 4)."""
    return (1.0 + 3.0 * -(-d // 8)) * 2.0 ** -20 * np.sqrt(nrm_i * nrm_j)


def tf32_rna(v):
    """cvt.rna.tf32.f32: round to the nearest 10-bit mantissa, ties away from zero."""
    b = np.asarray(v, dtype=np.float32).view(np.uint32)
    return ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def emulate_3xtf32(a, b, truncate=False):
    """g for row pairs (a[p], b[p]) as the wgmma chain forms it: hi = rna(x), lo = rna(x - hi); per k-block of 8 three
    MMAs (hi hi', hi lo', lo hi') each adding its 8 exact products to the fp32 accumulator with one rounding (to nearest,
    or toward zero with truncate=True)."""
    a, b = np.asarray(a, dtype=np.float32), np.asarray(b, dtype=np.float32)
    ah, bh = tf32_rna(a), tf32_rna(b)
    al, bl = tf32_rna(a - ah), tf32_rna(b - bh)
    d = a.shape[1]
    acc = np.zeros(a.shape[0], dtype=np.float32)

    def rnd(v):
        f = v.astype(np.float32)
        if truncate:
            over = np.abs(f.astype(np.float64)) > np.abs(v)
            f = np.where(over, np.nextafter(f, np.float32(0)), f)
        return f

    for k0 in range(0, d, 8):
        sl = slice(k0, min(d, k0 + 8))
        for x, y in ((ah, bh), (ah, bl), (al, bh)):
            acc = rnd(acc.astype(np.float64) + (x[:, sl].astype(np.float64) * y[:, sl].astype(np.float64)).sum(axis=1))
    return acc
