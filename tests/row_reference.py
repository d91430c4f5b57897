"""float64 restatement of the streaming row kernels (alq_score.cu: K1 scores, K2 BADGE factors, K2p pooled embedding,
row norms; alq_mase.cu: K6 MASE margins) and per-row error bounds derived from the kernels' fp32 arithmetic.  NumPy
only, no torch arithmetic: the CPU tier checks it against the torch oracle and scipy, the GPU tier checks the kernels
against it.

Error model shared by the bounds (u = 2^-24, gamma(k) = k u / (1 - k u), the standard bound of k rounded additions):

* exp term.  The kernels evaluate exp(d), d = z - max <= 0, as ex2.approx.ftz(fl(fl(z - max) * fl32(log2 e))).  The
  three roundings perturb the exponent by at most |d| ((1 + u)^3 - 1) and ex2.approx adds 2^-22 relative, so
      eta(d) = (1 + 2^-22) exp(3.01 u |d|) - 1           (relative error of one term; |d| capped at 104).
  Results below 2^-126 flush to zero: an absolute slack of c 2^-125 on the sum (and c 2^-125 * 104 on the entropy's
  sum of e d) covers every flushed term.
* sums.  The vector kernels add 4 ceil(c / 128) terms per lane in sequence and then 5 shuffle levels; the generic
  kernels ceil(c / 32) + 5.  A sum of terms t_j with depth k is within gamma(k) sum |t_j| of the exact sum of the
  computed terms.
* divisions, products, subtractions: one rounding u each; logf: 1 ulp <= 2 u |log s|.

With S = sum_j e_j and Es the bound on |s_hat - S|, rho = Es / S:
    least confidence  p1 = 1 / S:            p1 ((1 + u) / (1 - rho) - 1)
    margin            p1 - p2, p2 = e2 / S:  p1 ((1 + u) / (1 - rho) - 1) + p2 ((1 + eta2)(1 + u) / (1 - rho) - 1)
                                             + u (p1 + p2)
    entropy           W / S - log S, W = sum e_j d_j:  Ew / (S (1 - rho)) + |W / S| rho / (1 - rho)  (the quotient)
                                             + rho / (1 - rho) + 2 u |log S|  (the log)  + u per rounding of the two
                                             results and of their difference,
    Ew = sum e_j |d_j| ((1 + eta_j)(1 + u) - 1) + gamma(k) sum e_j |d_j| (1 + eta_j)(1 + u) + flush slack.
"""
import numpy as np

from oracle import al_oracle as O

MODE_MARGIN, MODE_LEAST_CONFIDENCE, MODE_ENTROPY = 0, 1, 2
U = 2.0 ** -24
EX2_REL = 2.0 ** -22
FLUSH = 2.0 ** -125                 # twice the smallest normal float: a term ex2.approx.ftz may flush to zero
D_CAP = 104.0                       # exp(-104) is far below the flush threshold: larger gaps change nothing
F32_OVERFLOW = 2.0 ** 128 - 2.0 ** 103     # the smallest real that rounds to +inf in fp32


def gamma(k):
    k = np.asarray(k, dtype=np.float64)
    return k * U / (1.0 - k * U)


def sum_depth(c, route):
    """Rounded additions on the longest path of a row sum: 'vec' (direct vector and pipelined kernels) or 'generic'."""
    if route == "vec":
        return 4 * -(-c // 128) + 5
    if route == "generic":
        return -(-c // 32) + 5
    raise ValueError(route)


def _parts(z):
    """(max, d = z - max, e = exp(d), S = sum e, bad rows) in float64; bad rows (a NaN or +inf logit, or every logit
    -inf) give NaN scores."""
    z = np.asarray(z, dtype=np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        m = z.max(axis=1)
        bad = ~np.isfinite(m)
        mm = np.where(bad, 0.0, m)
        d = z - mm[:, None]
        d[bad] = 0.0
        e = np.exp(d)
    return m, d, e, e.sum(axis=1), bad


def _eta(d):
    return (1.0 + EX2_REL) * np.exp(3.01 * U * np.minimum(np.abs(d), D_CAP)) - 1.0


def second_largest(z):
    """The second largest logit of every row counted with multiplicity (== the max when the max is repeated)."""
    z = np.asarray(z, dtype=np.float64)
    if z.shape[1] < 2:
        return np.full(z.shape[0], -np.inf)
    return -np.partition(-z, 1, axis=1)[:, 1]


def softmax_scores64(z, mode):
    """K1's scores in float64: margin p1 - p2 (p2 = p1 when the max is repeated), least confidence p1, entropy
    sum p log p with 0 log 0 = 0.  NaN for rows with a NaN or +inf logit or with every logit -inf (as torch)."""
    m, d, e, S, bad = _parts(z)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        if mode == MODE_MARGIN:
            t2 = second_largest(np.where(bad[:, None], 0.0, z))
            out = (1.0 - np.exp(t2 - np.where(bad, 0.0, m))) / S
        elif mode == MODE_LEAST_CONFIDENCE:
            out = 1.0 / S
        elif mode == MODE_ENTROPY:
            p = e / S[:, None]
            logp = d - np.log(S)[:, None]
            out = np.where(p == 0, 0.0, p * logp).sum(axis=1)
        else:
            raise ValueError(mode)
    out[bad] = np.nan
    return out


def score_bound(z, mode, route):
    """Per-row bound on |kernel score - softmax_scores64| (formula: module docstring).  NaN on the NaN rows."""
    z = np.asarray(z, dtype=np.float64)
    c = z.shape[1]
    m, d, e, S, bad = _parts(z)
    k = sum_depth(c, route)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        eta = _eta(d)
        Es = (e * eta).sum(1) + gamma(k) * (e * (1 + eta)).sum(1) + c * FLUSH
        rho = Es / S
        q = 1.0 / (1.0 - rho)
        p1 = 1.0 / S
        if mode == MODE_LEAST_CONFIDENCE:
            b = p1 * ((1 + U) * q - 1)
        elif mode == MODE_MARGIN:
            d2 = second_largest(np.where(bad[:, None], 0.0, z)) - np.where(bad, 0.0, m)
            e2 = np.exp(d2)
            p2 = e2 / S
            b = p1 * ((1 + U) * q - 1) + p2 * ((1 + _eta(d2)) * (1 + U) * q - 1) + FLUSH / S + U * (p1 + p2) * (1 + 4 * U)
        elif mode == MODE_ENTROPY:
            ad = np.abs(d)
            ed = np.where(e == 0, 0.0, e * ad)
            W = -ed.sum(1)
            Ew = (ed * ((1 + eta) * (1 + U) - 1)).sum(1) + gamma(k) * (ed * (1 + eta) * (1 + U)).sum(1) + c * FLUSH * D_CAP
            quo = np.abs(W) / S
            e_quo = Ew / S * q + quo * rho * q
            e_quo += U * (quo + e_quo)
            logS = np.log(S)
            e_log = rho * q + 2 * U * (logS + rho * q)
            b = e_quo + e_log + U * (quo + e_quo + logS + e_log)
        else:
            raise ValueError(mode)
    b = np.asarray(b, dtype=np.float64)
    b[bad] = np.nan
    return b


def batch_sizes(n, bs, row0=0, n_total=0):
    """Size of the loader batch each row [row0, row0 + n) of a pass over n_total rows falls in."""
    if not n_total:
        n_total, row0 = n, 0
    g = np.arange(row0, row0 + n)
    tail = n_total % bs
    return np.where((tail > 0) & (g >= n_total - tail), tail, bs).astype(np.float64)


def badge_factors64(z, bs, row0=0, n_total=0):
    """K2: a = (softmax(z) - onehot(first arg-max)) / (size of the row's loader batch), and |a|^2, in float64.
    Rows with a NaN or +inf logit, or every logit -inf, are NaN."""
    z = np.asarray(z, dtype=np.float64)
    m, d, e, S, bad = _parts(z)
    with np.errstate(invalid="ignore"):
        p = e / S[:, None]
        p[np.arange(len(p)), np.argmax(np.where(bad[:, None], 0.0, z), axis=1)] -= 1.0
        a = p / batch_sizes(z.shape[0], bs, row0, n_total)[:, None]
    a[bad] = np.nan
    return a, (a * a).sum(1)


def badge_bound(z, bs, route, row0=0, n_total=0):
    """(per-element bound on a, per-row bound on |a|^2) of K2.  p_j = e_j * fl(1 / s) (vector) or e_j / s (generic):
    two roundings at most; then p_j - onehot (u), times fl(1 / bs_i) (two roundings); the norm is a row sum of
    depth sum_depth(c, route) of rounded squares."""
    z = np.asarray(z, dtype=np.float64)
    c = z.shape[1]
    a, _ = badge_factors64(z, bs, row0, n_total)
    m, d, e, S, bad = _parts(z)
    k = sum_depth(c, route)
    bsz = batch_sizes(z.shape[0], bs, row0, n_total)[:, None]
    with np.errstate(invalid="ignore", over="ignore"):
        eta = _eta(d)
        Es = (e * eta).sum(1) + gamma(k) * (e * (1 + eta)).sum(1) + c * FLUSH
        q = (1.0 / (1.0 - Es / S))[:, None]
        p = e / S[:, None]
        err_p = p * ((1 + eta) * (1 + U) ** 2 * q - 1) + FLUSH / S[:, None]
        v = np.abs(a) * bsz
        err_v = err_p + U * (v + err_p)
        eg = (err_v * (1 + U) ** 2 + v * ((1 + U) ** 2 - 1)) / bsz
        ag = np.abs(a)
        en = ((2 * ag * eg + eg * eg) * (1 + U)).sum(1) + gamma(k + 1) * ((ag + eg) ** 2).sum(1)
    eg[bad] = np.nan
    en[bad] = np.nan
    return eg, en


def pooled64(z, h, bs):
    """K2p: the reference's adaptive-pooled gradient embedding, as the outer product of the 1-D pools of a (ph bins
    over the classes) and h (pw bins over the embedding), ph = min(16, c), pw = 512 // ph; [n, ph * pw] float64."""
    a, _ = badge_factors64(z, bs)
    h = np.asarray(h, dtype=np.float64)
    c, dd = a.shape[1], h.shape[1]
    ph = min(O.POOLING_H, c)
    pw = O.POOLING_AREA // ph
    pa = np.stack([a[:, lo:hi].mean(1) for lo, hi in O.adaptive_pool_bins(c, ph)], axis=1)
    phh = np.stack([h[:, lo:hi].mean(1) for lo, hi in O.adaptive_pool_bins(dd, pw)], axis=1)
    return (pa[:, :, None] * phh[:, None, :]).reshape(a.shape[0], -1)


def pooled_bound(z, h, bs):
    """Bound on |K2p - pooled64|: the factor of each class bin is K2's generic-route element (badge_bound) summed in
    sequence and divided by the bin width, the embedding bin likewise; their product is rounded once."""
    a, _ = badge_factors64(z, bs)
    eg, _ = badge_bound(z, bs, "generic")
    h = np.asarray(h, dtype=np.float64)
    c, dd = a.shape[1], h.shape[1]
    ph = min(O.POOLING_H, c)
    pw = O.POOLING_AREA // ph
    pa, epa, phh, eph = [], [], [], []
    for lo, hi in O.adaptive_pool_bins(c, ph):
        w = hi - lo
        s = np.abs(a[:, lo:hi].mean(1))
        e = (eg[:, lo:hi].sum(1) + gamma(w) * (np.abs(a[:, lo:hi]) + eg[:, lo:hi]).sum(1)) / w
        pa.append(s)
        epa.append(e + U * (s + e))
    for lo, hi in O.adaptive_pool_bins(dd, pw):
        w = hi - lo
        s = np.abs(h[:, lo:hi].mean(1))
        e = gamma(w) * np.abs(h[:, lo:hi]).sum(1) / w
        phh.append(s)
        eph.append(e + U * (s + e))
    pa, epa, phh, eph = (np.stack(t, axis=1) for t in (pa, epa, phh, eph))
    A, EA, H, EH = pa[:, :, None], epa[:, :, None], phh[:, None, :], eph[:, None, :]
    b = EA * H + A * EH + EA * EH + U * (A + EA) * (H + EH)
    return b.reshape(a.shape[0], -1)


def row_norm2_64(x):
    x = np.asarray(x, dtype=np.float64)
    return (x * x).sum(1)


def row_norm2_bound(x, vec):
    """Row sum of d rounded squares, depth 4 ceil(d / 128) + 5 (vector) or ceil(d / 32) + 5 (scalar): gamma(depth + 1)
    times the exact sum."""
    d = np.asarray(x).shape[1]
    return gamma(sum_depth(d, "vec" if vec else "generic") + 1) * row_norm2_64(x)


def gap_inv64(w):
    """1 / |w_a - w_c| in float64, +inf on the diagonal and where class rows coincide."""
    w = np.asarray(w, dtype=np.float64)
    den = ((w[:, None, :] - w[None, :, :]) ** 2).sum(2)
    with np.errstate(divide="ignore"):
        g = 1.0 / np.sqrt(den)
    np.fill_diagonal(g, np.inf)
    return g


def mase64(z, w):
    """K6's closed form in float64: pred = torch.max's arg-max (the first maximum; the first NaN in a row with a NaN),
    radius[i, c] = |z_ip - z_ic| / |w_p - w_c| with NaN -> +inf and radius[i, p] = +inf, min_margin = the row minimum.
    The logit gap and the radius are float32 quantities in the reference too: values that round to +inf in fp32
    are +inf here.  Returns (min_margin, pred, radius)."""
    z = np.asarray(z, dtype=np.float64)
    n, c = z.shape
    pred = np.argmax(z, axis=1)                       # NumPy's argmax also returns the first NaN
    g = gap_inv64(w)
    with np.errstate(invalid="ignore", over="ignore"):
        gap = np.abs(z[np.arange(n), pred][:, None] - z)
        gap = np.where(gap >= F32_OVERFLOW, np.inf, gap)
        r = gap * g[pred]
    r = np.where(np.isnan(r) | (r >= F32_OVERFLOW), np.inf, r)
    r[np.arange(n), pred] = np.inf
    return r.min(1), pred, r


def mase_bound(radius, m):
    """Relative bound of K6's radii: the fp32 gap and the product (two roundings) and the fp32 table 1 / |w_p - w_c|
    (m rounded squares of rounded differences summed by fma, sqrt, reciprocal: gamma(m + 6))."""
    rel = (1 + U) ** 2 * (1 + gamma(m + 6)) - 1
    with np.errstate(invalid="ignore"):
        return np.where(np.isfinite(radius), radius * rel, 0.0)
