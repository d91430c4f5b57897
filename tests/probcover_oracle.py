"""NumPy statement of ProbCoverSampler's query (active_learning_b200/query_strategies/probcover.py, kernels K13 / K14),
written from the algorithm of Yehuda et al., "Active Learning Through a Covering Lens" (NeurIPS 2022):

  normalise  lane l of 32 sums the fp64 squares of columns l, l + 32, .. in order, a butterfly (xor 16, 8, 4, 2, 1)
             adds the partials, norm = sqrt, xhat = fl32(x / norm) in fp64; a zero row stays zero;
  graph      an edge (i, j) iff scipy's fp64 euclidean distance of xhat_i, xhat_j is < delta (d = a - b, s = s + d * d,
             k ascending, then sqrt), as CSR with ascending columns;
  greedy     covered = the balls of the labeled rows; deg[x] = uncovered rows in N(x); each step stops if max deg = 0,
             else takes the lowest position c of the maximum and covers N(c);
  fill       the rest of the budget is np.random.choice(available-and-unpicked positions ascending, rest, replace=False).

The tensor-core screen's pieces (DESIGN section 4) follow: its bound E, its band decision in the epilogue's fp64
order, emulations of the 3xTF32 chain under three adder models, and rows that stress E.
"""
import math

import numpy as np

LANES = 32


def lane_sum_sq(x):
    """K13's fp64 sum of squares of each fp32 row: lane l of 32 adds the squares of columns l, l + 32, .. in order, then a
    butterfly (xor 16, 8, 4, 2, 1) adds the 32 partials."""
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
    return s[:, 0]


def nrm2(xhat):
    """K13's nrm2_i = |xhat_i|^2 in fp64, the order of lane_sum_sq."""
    return lane_sum_sq(xhat)


def normalize(x):
    x = np.asarray(x, dtype=np.float32)
    n, d = x.shape
    norm = np.sqrt(lane_sum_sq(x))
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


EDGE, NONE, RECHECK = 1, 0, 2


def screen_decide(d, ni, nj, g, delta):
    """The epilogue's decision for fp32 dot products g of rows with nrm2 ni, nj at width d (K13's padded width), in fp64
    and in the kernel's operation order: EDGE, NONE, or RECHECK (inside the band: the exact recomputation decides)."""
    coef = 2.0 * screen_bound(d, 1.0, 1.0) * (1.0 + 1e-6)
    delta2 = float(delta) * float(delta)
    slack = 1e-9 * delta2 + 1e-10
    ni, nj = np.asarray(ni, dtype=np.float64), np.asarray(nj, dtype=np.float64)
    d2 = (ni + nj) - 2.0 * np.asarray(g, dtype=np.float32).astype(np.float64)
    bnd = coef * np.sqrt(ni * nj) + slack
    return np.where(d2 < delta2 - bnd, EDGE, np.where(d2 > delta2 + bnd, NONE, RECHECK))


def _to_f32_toward_zero(v):
    f = v.astype(np.float32)
    over = np.abs(f.astype(np.float64)) > np.abs(v)
    return np.where(over, np.nextafter(f, np.float32(0)), f)


def emulate_3xtf32(a, b, adder="nearest", bits=24):
    """g for row pairs (a[p], b[p]) as the wgmma chain forms it: hi = rna(x), lo = rna(x - hi); per k-block of 8 three
    MMAs (hi hi', hi lo', lo hi'), each adding its 8 exact products to the fp32 accumulator.  The adder of one MMA:
      "nearest"  the exact sum rounded once to nearest;
      "zero"     the exact sum rounded once toward zero;
      "align"    the accumulator and the 8 products aligned to the largest exponent among them, each truncated to `bits`
                 bits below and including that exponent's leading bit, summed exactly, the sum truncated to fp32."""
    a, b = np.asarray(a, dtype=np.float32), np.asarray(b, dtype=np.float32)
    ah, bh = tf32_rna(a), tf32_rna(b)
    al, bl = tf32_rna(a - ah), tf32_rna(b - bh)
    d = a.shape[1]
    acc = np.zeros(a.shape[0], dtype=np.float32)
    for k0 in range(0, d, 8):
        sl = slice(k0, min(d, k0 + 8))
        for x, y in ((ah, bh), (ah, bl), (al, bh)):
            prods = x[:, sl].astype(np.float64) * y[:, sl].astype(np.float64)
            if adder == "align":
                terms = np.concatenate([acc.astype(np.float64)[:, None], prods], axis=1)
                _, ex = np.frexp(np.max(np.abs(terms), axis=1))        # largest |term| in [2^(ex - 1), 2^ex)
                q = np.ldexp(1.0, ex - bits)[:, None]
                acc = _to_f32_toward_zero((np.trunc(terms / q) * q).sum(axis=1))    # exact: < 2^53 units of q
            else:
                s = acc.astype(np.float64) + prods.sum(axis=1)
                acc = s.astype(np.float32) if adder == "nearest" else _to_f32_toward_zero(s)
    return acc


# ---- rows that stress the bound -------------------------------------------------------------------------------------
def _low_bits(x, pattern):
    """x with the low 13 mantissa bits (those TF32 drops) set to `pattern`."""
    u = np.asarray(x, dtype=np.float32).view(np.uint32)
    return ((u & np.uint32(0xFFFFE000)) | np.uint32(pattern)).view(np.float32)


def bound_families(rng, d, instances=3):
    """{family: [m, d] float32 rows} of near-unit rows (normalize'd) at which the 3xTF32 chain's error is largest relative
    to E.  The TF32 bit patterns are imposed after normalisation, which moves |x|^2 by at most 2^-10."""
    k = np.arange(d)
    u = lambda: rng.random(d)                                              # noqa: E731
    sign = lambda: rng.choice([-1.0, 1.0], d)                              # noqa: E731
    raw = {
        "equal": [np.ones(d), -np.ones(d)],
        "full_mantissa": [1.0 + u() for _ in range(instances)],            # same sign: the accumulator dwarfs a product
        "midpoint": [1.0 + u() for _ in range(instances)],
        "below_midpoint": [(1.0 + u()) * sign() for _ in range(instances)],
        "spike_first": [], "spike_last": [],
        "alternating": [(-1.0) ** (k >> s) * (1.0 + 1e-3 * u()) for s in range(instances)],   # Walsh signs: S >> |g|
        "ramp": [2.0 ** (-4.0 * ((k + s) % 8) - 3.0 * k / max(d - 1, 1)) * (1.0 + u()) * sign() for s in range(instances)],
        "normal": [rng.normal(size=d) for _ in range(instances)],
        "abs_normal": [np.abs(rng.normal(size=d)) for _ in range(instances)],
    }
    for _ in range(instances):
        tiny = 1e-4 * (1.0 + u()) * sign()
        first, last = tiny.copy(), tiny.copy()
        first[0], last[-1] = 1.0, -1.0
        raw["spike_first"].append(first)
        raw["spike_last"].append(last)
    fam = {name: normalize(np.stack(rows).astype(np.float32)) for name, rows in raw.items()}
    fam["midpoint"] = _low_bits(fam["midpoint"], 0x1000)                  # on a midpoint: |lo| = half a TF32 ulp ...
    fam["below_midpoint"] = _low_bits(fam["below_midpoint"], 0x0FFF)      # ... just below: lo, and lo lo', at their largest
    base = np.concatenate(list(fam.values()))
    noise = (rng.normal(size=base.shape) * 1e-4).astype(np.float32)
    fam["near_duplicate"] = normalize(base + noise * np.abs(base).max(axis=1, keepdims=True))   # d^2 next to 0
    fam["antipode"] = -base
    return fam


def exact_dots(a, b):
    """<a_p, b_p> of fp32 rows correctly rounded to fp64: the products are exact in fp64, math.fsum adds them exactly."""
    a, b = np.asarray(a, dtype=np.float32).astype(np.float64), np.asarray(b, dtype=np.float32).astype(np.float64)
    return np.array([math.fsum(p) for p in a * b])
