"""NumPy statement of CALSampler's query (active_learning_b200/query_strategies/cal.py, kernels K18, K19, K1b), written
from Margatina, Vernikos, Barrault & Aletras, "Active Learning by Acquiring Contrastive Examples" (EMNLP 2021) and the
authors' selection loop.  Matching sklearn's fp32 k-NN distances or torch's fp32 KL divergence is not a goal (DESIGN
section 2).

  pool        CoreSet's union (two shuffles); the references R are its labeled rows (M), the candidates its available
              rows (N); the budget is min(budget, N), 0 returns nothing; M = 0 raises ValueError; no NumPy draw beyond the
              two shuffles;
  forward     one pool forward of the task network: fp32 logits z and embeddings (padded with zero columns);
  neighbours  k = min(NUM_NEIGHBORS, M); candidate i's k rows of R with the smallest exact_d2 (K7's pair arithmetic on the
              raw, unnormalised embeddings: d = a - b, s = s + d * d, ascending, no FMA, fp64), ties to the lower
              position in R; past M the entries are -1 / +inf;
  score       per row r in fp64: lse_r = m_r + log(sum_c exp(z_rc - m_r)), m_r = max_c z_rc, the sum in ascending c;
              lp_rc = z_rc - lse_r; p_rc = exp(lp_rc); KL(n || i) = sum_c p_nc (lp_nc - lp_ic) in ascending c;
              score_i = (sum_j KL(n_j || i)) / k, the neighbours in ascending (d2, position) order;
  picks       the budget largest fl32(score_i), lowest position on ties, in that order: K1b's ascending
              (alq_ord(key), position) on key = -fl32(score_i).  alq_ord puts -0.0 below +0.0, so a zero score's key is
              written +0.0 (else zero scores would not tie by position); a NaN score's key is +NaN and sorts last.

`authors_select` restates the authors' loop literally: sklearn's KNeighborsClassifier and one `kneighbors` per candidate,
torch fp32 softmax / log_softmax / KLDivLoss(reduction="none") summed over the classes, the mean over the neighbours,
np.argpartition for the top b.  `band` is K18's screen band, `screen_lower` its fp32 lower bounds in the kernel's order and
`fallback_decide` its fallback decision; `score_bound` is the bound on K19's distance from `scores` that CUDA's exp / log
allow (DESIGN section 4).
"""
import math

import numpy as np

import probcover_oracle as P

NUM_NEIGHBORS = 10
exact_d2 = P.exact_d2
U = 2.0 ** -53


# ---- K18: the exact k nearest rows ---------------------------------------------------------------------------------------
def knn(x, y, k):
    """(idx int64 [n, k], d2 fp64 [n, k]): per row of x the k rows of y with the smallest exact_d2, ascending (d2, row),
    -1 / +inf past len(y).  An fp64 GEMM screens the pairs; only the columns that can reach the k-th are computed
    exactly (the screen's error is far below 1e-9 (|x| + |y|)^2)."""
    x, y = np.asarray(x, dtype=np.float32), np.asarray(y, dtype=np.float32)
    n, m = x.shape[0], y.shape[0]
    x64, y64 = x.astype(np.float64), y.astype(np.float64)
    nx, ny = (x64 * x64).sum(1), (y64 * y64).sum(1)
    sx, sy = np.sqrt(nx), np.sqrt(ny)
    idx = np.full((n, k), -1, dtype=np.int64)
    d2 = np.full((n, k), np.inf)
    kk = min(k, m)
    for lo in range(0, n, 256):
        hi = min(n, lo + 256)
        scr = nx[lo:hi, None] + ny[None, :] - 2.0 * (x64[lo:hi] @ y64.T)
        tau = 1e-9 * (sx[lo:hi, None] + sy[None, :]) ** 2
        up = np.partition(scr + tau, kk - 1, axis=1)[:, kk - 1]
        ri, cj = np.nonzero(scr - tau <= up[:, None])
        ex = exact_d2(x[lo + ri], y[cj])
        for r in range(hi - lo):
            sel = ri == r
            e, j = ex[sel], cj[sel]
            o = np.lexsort((j, e))[:kk]
            idx[lo + r, :kk] = j[o]
            d2[lo + r, :kk] = e[o]
    return idx, d2


# ---- K19: the scores -------------------------------------------------------------------------------------------------------
def log_softmax(z):
    """(lse [r], lp [r, C]) in fp64 from fp32 logits: the max, the ascending sum of exp(z - max), its log."""
    z64 = np.asarray(z, dtype=np.float32).astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        m = z64.max(axis=1)
        s = np.cumsum(np.exp(z64 - m[:, None]), axis=1)[:, -1]
        lse = m + np.log(s)
        return lse, z64 - lse[:, None]


def scores(cand_logits, ref_logits, idx):
    """score_i (fp64 [n]): the neighbours' KL(n || i) summed in list order over those in [0, M), divided by their number
    (0 when there is none)."""
    _, lpi = log_softmax(cand_logits)
    _, lpr = log_softmax(ref_logits)
    idx = np.asarray(idx, dtype=np.int64)
    n, k = idx.shape
    valid = (idx >= 0) & (idx < lpr.shape[0])
    out = np.zeros(n)
    for lo in range(0, n, 512):
        hi = min(n, lo + 512)
        lpn = lpr[np.where(valid[lo:hi], idx[lo:hi], 0)]                          # [r, k, C]
        with np.errstate(invalid="ignore", over="ignore"):
            t = np.exp(lpn) * (lpn - lpi[lo:hi, None, :])
            kl = np.where(valid[lo:hi], np.cumsum(t, axis=2)[..., -1], 0.0)      # a skipped neighbour adds +0.0
            cnt = valid[lo:hi].sum(1)
            s = np.cumsum(kl, axis=1)[:, -1]
            out[lo:hi] = np.where(cnt > 0, s / np.maximum(cnt, 1), 0.0)
    return out


def keys(score):
    """K1b's key: -fl32(score), +0.0 for a zero and +NaN for a NaN score."""
    f = np.asarray(score, dtype=np.float64).astype(np.float32)
    key = np.where(f == 0, np.float32(0.0), -f).astype(np.float32)
    return np.where(np.isnan(score), np.float32(np.nan), key).astype(np.float32)


def alq_ord(key):
    u = np.asarray(key, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return np.where(u & 0x80000000, (~u) & 0xFFFFFFFF, u | 0x80000000)


def select(key, budget):
    """Positions of the budget smallest keys in ascending (alq_ord(key), position) order."""
    return np.lexsort((np.arange(len(key)), alq_ord(key)))[:int(budget)].astype(np.int64)


def query_positions(emb, logits, is_lab, avail, budget):
    """Positions in the pool that the query returns, in order."""
    budget = int(min(int(np.sum(avail)), budget))
    if budget <= 0:
        return np.zeros(0, dtype=np.int64)
    lab, cand = np.flatnonzero(is_lab), np.flatnonzero(avail)
    if not len(lab):
        raise ValueError("CALSampler needs labeled rows")
    k = min(NUM_NEIGHBORS, len(lab))
    emb, logits = np.asarray(emb, dtype=np.float32), np.asarray(logits, dtype=np.float32)
    idx, _ = knn(emb[cand], emb[lab], k)
    return cand[select(keys(scores(logits[cand], logits[lab], idx)), budget)]


# ---- the authors' loop ---------------------------------------------------------------------------------------------------
def authors_select(emb_lab, logits_lab, emb_cand, logits_cand, budget, k=NUM_NEIGHBORS):
    """The authors' CAL selection restated literally: positions into the candidates (a set: np.argpartition's order)."""
    import torch
    import torch.nn.functional as F
    from sklearn.neighbors import KNeighborsClassifier
    neigh = KNeighborsClassifier(n_neighbors=k)
    neigh.fit(X=emb_lab, y=np.zeros(len(emb_lab), dtype=np.int64))
    criterion = torch.nn.KLDivLoss(reduction="none")
    train_logits = torch.from_numpy(np.asarray(logits_lab, dtype=np.float32))
    kl_scores = []
    for i in range(len(emb_cand)):
        neighbours = neigh.kneighbors(X=[emb_cand[i]], return_distance=False)
        neigh_prob = F.softmax(train_logits[neighbours], dim=-1)
        candidate_log_prob = F.log_softmax(torch.from_numpy(np.asarray(logits_cand[i], dtype=np.float32)), dim=-1)
        kl = np.array([torch.sum(criterion(candidate_log_prob, n), dim=-1).numpy() for n in neigh_prob])
        kl_scores.append(kl.mean())
    return np.argpartition(np.asarray(kl_scores), -budget)[-budget:]


# ---- K18's band ----------------------------------------------------------------------------------------------------------
def band(d, nrm_i, nrm_j):
    """K18's half-width b >= |d2~ - exact_d2| for rows of squared norms nrm_i, nrm_j at padded width d (DESIGN section 4)."""
    si, sj = np.sqrt(np.asarray(nrm_i, dtype=np.float64)), np.sqrt(np.asarray(nrm_j, dtype=np.float64))
    coef = 2.0 * P.screen_bound(d, 1.0, 1.0) * (1.0 + 1e-6)
    t = si + sj
    return coef * (si * sj) + (4.0 * d + 32.0) * U * (t * t) + d * 2.0 ** -100 * (1.0 + t)


def _f32_down(v):
    """fp64 values rounded down to fp32 (__double2float_rd): NumPy rounds to nearest, so step down where that lands
    above the fp64 value."""
    v = np.asarray(v, dtype=np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        f = v.astype(np.float32)
        return np.where(f.astype(np.float64) > v, np.nextafter(f, np.float32(-np.inf)), f).astype(np.float32)


def screen_lower(d, nrm_i, nrm_j, g):
    """K18's lower bounds L [.., ..] float32 for fp32 dot products g of rows with squared norms nrm_i, nrm_j (their
    lane-ordered fp64 values) at width d, as knn_screen_kernel forms them: d2~ = (nrm_i + nrm_j) - 2 g,
    t = sqrt(nrm_i) + sqrt(nrm_j), b = (coef (sx sy) + rel (t t)) + abs (1 + t), fl32_down(d2~ - b)."""
    ni, nj = np.asarray(nrm_i, dtype=np.float64), np.asarray(nrm_j, dtype=np.float64)
    sx, sy = np.sqrt(ni), np.sqrt(nj)
    coef = 2.0 * P.screen_bound(d, 1.0, 1.0) * (1.0 + 1e-6)
    rel, abs_ = (4.0 * d + 32.0) * U, d * 2.0 ** -100
    t = sx + sy
    b = (coef * (sx * sy) + rel * (t * t)) + abs_ * (1.0 + t)
    return _f32_down(screen_d2(ni, nj, g) - b)


S_KEPT = 32                            # lower bounds K18 keeps per row


def fallback_decide(L, exact, k):
    """K18's fallback decision per row of the lower bounds L [n, m]: the kept set is the S_KEPT smallest L, L* the
    (S_KEPT + 1)-th smallest (+inf for m <= S_KEPT), E_k the k-th exact d2 over the kept columns in (d2, column) order,
    and the row falls back iff L* <= E_k.  `exact(rows, cols)` gives exact_d2 for index pairs; it is called only for the
    kept columns and those tied with the last kept bound.  Returns, per row, the frozenset of decisions the kernel can
    reach: two only when L ties across the boundary and the kept set changes the decision, which needs a bound above its
    exact value (a tied column at or above L* never sets E_k below L*)."""
    L = np.asarray(L, dtype=np.float32)
    n, m = L.shape
    if m <= S_KEPT:
        return [frozenset([False])] * n
    order = np.argsort(L, axis=1, kind="stable")
    srt = np.take_along_axis(L, order, axis=1)
    lstar = srt[:, S_KEPT]
    edge = srt[:, S_KEPT - 1]
    # the columns certainly kept (below the last kept bound) and the candidates for the rest (tied with it)
    rows, cols = [], []
    for i in range(n):
        c = np.flatnonzero(L[i] <= edge[i]) if lstar[i] == edge[i] else order[i, :S_KEPT]
        rows.append(np.full(len(c), i))
        cols.append(c)
    ex = exact(np.concatenate(rows), np.concatenate(cols))
    out, at = [], 0
    for i in range(n):
        c = cols[i]
        e = ex[at:at + len(c)]
        at += len(c)
        if np.isinf(lstar[i]):
            out.append(frozenset([False]))
            continue
        sure = L[i, c] < edge[i]
        need = S_KEPT - int(sure.sum())            # kept from the tied columns
        o = np.lexsort((c[~sure], e[~sure]))
        tied_e, tied_c = e[~sure][o], c[~sure][o]
        dec = set()
        for pick in (slice(0, need), slice(len(tied_c) - need, len(tied_c))):   # the smallest and the largest E_k
            ke, kc = np.concatenate([e[sure], tied_e[pick]]), np.concatenate([c[sure], tied_c[pick]])
            ek = ke[np.lexsort((kc, ke))][k - 1]
            dec.add(bool(float(lstar[i]) <= ek))
        out.append(frozenset(dec))
    return out


def screen_d2(nrm_i, nrm_j, g):
    """d2~ = (nrm2_i + nrm2_j) - 2 g in fp64, the epilogue's order."""
    return (np.asarray(nrm_i, dtype=np.float64) + np.asarray(nrm_j, dtype=np.float64)) - 2.0 * np.asarray(
        g, dtype=np.float32).astype(np.float64)


# ---- K19's distance from `scores` -----------------------------------------------------------------------------------------
ULPS = 4                               # exp / log within 4 ulp of the real value, on either side (CUDA: 1; NumPy: <= 4)


def score_bound(cand_logits, ref_logits, idx, score):
    """Per candidate, a bound on |K19's score - scores()| when both follow the same operation order and differ only in
    exp / log, each within ULPS ulp (DESIGN section 4)."""
    q = 2.0 * ULPS * U                                  # a relative error of ULPS ulp
    lse_c, lpi = log_softmax(cand_logits)
    lse_r, lpr = log_softmax(ref_logits)
    C = lpi.shape[1]

    def delta(lse, lp):                                 # |lp_dev - lp_oracle| per row
        a = np.abs(lp).max(axis=1)
        return 1.05 * (2 * q + 2 * (C + 2) * U + 2 * q * math.log(max(C, 2)) + 4 * U * np.abs(lse) + 4 * U * a), a
    dc, ac = delta(lse_c, lpi)
    dr, ar = delta(lse_r, lpr)
    idx = np.asarray(idx, dtype=np.int64)
    valid = (idx >= 0) & (idx < lpr.shape[0])
    nb = np.where(valid, idx, 0)
    A = ar[nb] + ac[:, None]                            # |lp_n - lp_i| <= A
    beta = 1.05 * ((dr[nb] + 2 * q + 4 * U) * A + dr[nb] + dc[:, None]) + 2.1 * C * U * A
    beta = np.where(valid, beta, 0.0)
    cnt = np.maximum(valid.sum(1), 1)
    return 1.05 * (beta.sum(1) + 2 * cnt * U * cnt * np.abs(score)) / cnt + 4 * U * np.abs(score)
