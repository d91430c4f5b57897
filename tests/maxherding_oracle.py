"""NumPy statement of MaxHerdingSampler's query (active_learning_b200/query_strategies/maxherding.py, kernels K22 / K23),
written from the algorithm of Bae, Noh & Sutherland, "Generalized Coverage for More Robust Low-Budget Active Learning"
(ECCV 2024):

  normalise  xhat = probcover_oracle.normalize(emb) (Engine.normalize);
  kernel     s_ij = probcover_oracle.exact_d2(xhat_i, xhat_j) (K7's fp64 chain: k ascending, no FMA) and
             K_ij = fl32(exp(-(s_ij / q))), q = 2 sigma^2 formed once in fp64 (herding_q); K is exactly symmetric and its
             diagonal is 1;
  objective  F(S) = sum_i max_{s in L u S} K_is over every row i of the pool, labeled rows included;
  greedy     m_i = max_{l in L} K_li (0.0f with L empty); gain_c = sum_{i ascending} max(0, K_ic - m_i) in fp64.  Each step
             takes c* = the lowest available, unpicked position of the largest gain, S = the ascending rows i with
             K[c*, i] > m_i, gain_c -= sum_{i in S ascending} (max(0, K_ic - m_i) - max(0, K_ic - K[c*, i])) for every
             column c, then m_i = K[c*, i] on S; min(budget, #available) steps.  No NumPy draw after the pool's shuffles.

`literal_greedy` recomputes every gain F(S u {c}) - F(S) from the matrix at every step (exactly rounded: math.fsum).
"""
import math
import sys

import numpy as np

import probcover_oracle as P

normalize = P.normalize


def herding_q(sigma):
    """q = 2 sigma^2 in fp64, as maxherding.herding_q forms it: ValueError unless sigma is finite and > 0 and q is a
    finite positive normal number."""
    if sigma is None:
        raise ValueError("sigma is required")
    sigma = float(sigma)
    if not (math.isfinite(sigma) and sigma > 0):
        raise ValueError(f"sigma must be finite and > 0, got {sigma}")
    q = 2.0 * sigma * sigma
    if not (math.isfinite(q) and q >= sys.float_info.min):
        raise ValueError(f"2 sigma^2 = {q} is not a finite positive normal number")
    return q


def d2_block(xhat, rows, cols=None):
    """exact_d2 of every (rows[a], cols[b]) pair as an [len(rows), len(cols)] fp64 block: k ascending, no FMA."""
    x = np.asarray(xhat, dtype=np.float32)
    a = x[np.asarray(rows)].astype(np.float64)
    b = x if cols is None else x[np.asarray(cols)]
    b = b.astype(np.float64)
    s = np.zeros((a.shape[0], b.shape[0]))
    for k in range(x.shape[1]):
        df = a[:, k, None] - b[None, :, k]
        s = s + df * df
    return s


def kernel_rows(xhat, q, rows):
    """Rows `rows` of the kernel matrix (fp32 [len(rows), n]) and their fp64 values before the fl32 rounding."""
    e = np.exp(-(d2_block(xhat, rows) / q))
    return e.astype(np.float32), e


def kernel_matrix(xhat, q, block=256):
    n = xhat.shape[0]
    out = np.empty((n, n), dtype=np.float32)
    for lo in range(0, n, block):
        out[lo:lo + block] = kernel_rows(xhat, q, np.arange(lo, min(n, lo + block)))[0]
    return out


def f32_midpoint_band(e):
    """Entries whose fp64 value e lies within 1 fp64 ulp of an fp32 rounding midpoint: CUDA's exp is within 1 ulp, so
    only there may fl32 of it differ from fl32 of NumPy's (by one fp32 ulp)."""
    e = np.asarray(e, dtype=np.float64)
    f = e.astype(np.float32)
    lo = np.where(f.astype(np.float64) <= e, f, np.nextafter(f, np.float32(-np.inf)))
    hi = np.nextafter(lo, np.float32(np.inf))
    mid = (lo.astype(np.float64) + hi.astype(np.float64)) / 2.0          # exact: fp32 neighbours
    return np.abs(e - mid) <= np.spacing(np.abs(e))


def initial_m(K, labeled):
    lab = np.flatnonzero(labeled)
    if len(lab) == 0:
        return np.zeros(K.shape[0], dtype=np.float32)
    return K[lab].max(axis=0)


def _seq_sum_rows(acc, terms):
    """acc + terms[0] + terms[1] + ..., sequentially (np.cumsum is a left-to-right loop)."""
    return np.cumsum(np.concatenate([acc[None], terms]), axis=0)[-1]


def greedy(K, labeled, avail, budget, block=256, return_gains=False):
    """The incremental greedy: (picks int64 in pick order, final m fp32[, gains before each pick as a list])."""
    K = np.asarray(K, dtype=np.float32)
    n = K.shape[0]
    m = initial_m(K, labeled)
    m64 = m.astype(np.float64)
    gain = np.zeros(n)
    for lo in range(0, n, block):
        gain = _seq_sum_rows(gain, np.maximum(0.0, K[lo:lo + block].astype(np.float64) - m64[lo:lo + block, None]))
    cand = np.asarray(avail, dtype=bool).copy()
    steps = int(min(int(budget), int(cand.sum())))
    picks, seen = [], []
    for _ in range(steps):
        if return_gains:
            seen.append(gain.copy())
        c = int(np.argmax(np.where(cand, gain, -np.inf)))
        kc = K[c]
        S = np.flatnonzero(kc > m)
        acc = np.zeros(n)
        for lo in range(0, len(S), block):
            rows = S[lo:lo + block]
            Kr = K[rows].astype(np.float64)
            t1 = np.maximum(0.0, Kr - m[rows].astype(np.float64)[:, None])
            t2 = np.maximum(0.0, Kr - kc[rows].astype(np.float64)[:, None])
            acc = _seq_sum_rows(acc, t1 - t2)
        gain = gain - acc
        m[S] = kc[S]
        cand[c] = False
        picks.append(c)
    picks = np.asarray(picks, dtype=np.int64)
    return (picks, m, seen) if return_gains else (picks, m)


def literal_gains(K, m, cols):
    """F(S u {c}) - F(S) for each c in cols, from the matrix, exactly rounded."""
    m64 = np.asarray(m, dtype=np.float64)
    return np.array([math.fsum(np.concatenate([np.maximum(m64, K[:, c].astype(np.float64)), -m64])) for c in cols])


def literal_greedy(K, labeled, avail, budget):
    """The greedy restated literally: every step recomputes F(S u {c}) - F(S) for every candidate and takes the lowest
    position of the largest.  Returns (picks, the gains of every step as {position: gain})."""
    K = np.asarray(K, dtype=np.float32)
    m = initial_m(K, labeled)
    cand = np.asarray(avail, dtype=bool).copy()
    picks, gains = [], []
    for _ in range(int(min(int(budget), int(cand.sum())))):
        cols = np.flatnonzero(cand)
        g = literal_gains(K, m, cols)
        c = int(cols[int(np.argmax(g))])
        gains.append(dict(zip(cols.tolist(), g.tolist())))
        m = np.maximum(m, K[c])
        cand[c] = False
        picks.append(c)
    return np.asarray(picks, dtype=np.int64), gains


def query_positions(emb, is_lab, avail, budget, sigma):
    """Positions in the pool that the query returns, in pick order."""
    budget = int(min(int(np.sum(avail)), budget))
    if budget <= 0:
        return np.zeros(0, dtype=np.int64)
    K = kernel_matrix(normalize(emb), herding_q(sigma))
    return greedy(K, is_lab, avail, budget)[0]
