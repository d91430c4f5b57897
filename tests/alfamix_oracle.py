"""NumPy statement of ALFAMixSampler's query (active_learning_b200/query_strategies/alfamix.py, kernels K16, K20, K5, K15,
K21), written from Parvaneh et al., "Active Learning by Feature Mixing" (CVPR 2022) with the algebra of the closed-form
alpha carried out.  Everything is fp64 in a fixed operation order; K20 follows it operation for operation and differs only
through CUDA's exp / log (`rho_bound`).

  pool       CoreSet's union (two shuffles); the candidates are its available rows, the budget is clamped to them, 0
             returns nothing; no labeled row raises ValueError;
  anchors    a_c = the fl32 mean of the labeled embeddings of class c (typiclust_oracle.update: the fp64 sequential sum in
             row order / m), a class without labeled rows the fl32 mean of all labeled rows;
  rho        G = W W^T (an ascending-d chain per entry); per row lse as cal_oracle.log_softmax, yhat = argmax l (lowest),
             r = exp(l - lse) - e_yhat; w = sum_c r_c G[c] (c ascending); s2 = sum_k r_k w_k (k ascending); t* = min over
             {k : w_k > w_yhat} of ((l_yhat - l_k) s) / (w_k - w_yhat), s = sqrt(s2), +inf when s2 <= 0 or no k;
             R2 = max_c exact_d2(z, a_c) (K7's pair arithmetic); rho = (sqrt(D) t*) / sqrt(R2), +inf when R2 = 0 or
             t* = +inf;
  caps       kappa_j = j * alpha_step (fp64), j = 1 .. ceil(1 / alpha_step); the candidate set {rho < kappa_j} of the
             first j that holds more than `budget` rows, else of the last j;
  diversity  no more candidates than the budget: all of them, ascending; otherwise typiclust_oracle's k-means of the
             normalised candidate rows with K = budget (one np.random.choice(|cand|), K - 1 np.random.random_sample, at
             most 100 assignments), and per non-empty cluster in id order the member with the smallest exact_d2 to its
             centre, the lowest position on ties;
  fill       probcover_oracle.random_fill over the available, unpicked rows.

`literal_flips` restates the paper's mixing literally (the per-coordinate alpha*, (1 - alpha*) z + alpha* a through an
fp64 nn.Linear, the argmax), for checking the collapse.
"""
import math

import numpy as np
import torch

import cal_oracle as CO
import probcover_oracle as P
import typiclust_oracle as T

U = 2.0 ** -53
ALPHA_STEP = 2.0 ** -5
MAX_ITER = 100


# ---- anchors -------------------------------------------------------------------------------------------------------------
def anchors(emb_lab, labels, num_classes):
    emb_lab = np.asarray(emb_lab, dtype=np.float32)
    mean = T.update(emb_lab, np.zeros(len(emb_lab), dtype=np.int64), np.zeros((1, emb_lab.shape[1]), dtype=np.float32))
    return T.update(emb_lab, np.asarray(labels, dtype=np.int64), np.repeat(mean, num_classes, axis=0))


# ---- K20 -----------------------------------------------------------------------------------------------------------------
def gram(weight):
    w = np.asarray(weight, dtype=np.float32).astype(np.float64)
    g = np.zeros((w.shape[0], w.shape[0]))
    for k in range(w.shape[1]):
        g = g + w[:, k, None] * w[None, :, k]
    return g


def residuals(logits):
    """(yhat [n], r [n, C]): the lowest argmax and p - e_yhat with p = exp(l - lse)."""
    z = np.asarray(logits, dtype=np.float32)
    lse, _ = CO.log_softmax(z)
    y = np.argmax(z, axis=1)
    r = np.exp(z.astype(np.float64) - lse[:, None])
    rows = np.arange(len(z))
    r[rows, y] = r[rows, y] - 1.0
    return y, r


def head_terms(logits, weight, g=None):
    """(yhat, r, w, s2): the per-row quantities of the head (w = G r, s2 = r^T w), in the spec's order."""
    g = gram(weight) if g is None else g
    y, r = residuals(logits)
    w = np.zeros_like(r)
    for c in range(r.shape[1]):
        w = w + r[:, c, None] * g[None, c, :]
    s2 = np.zeros(len(r))
    for k in range(r.shape[1]):
        s2 = s2 + r[:, k] * w[:, k]
    return y, r, w, s2


def tstar(logits, y, w, s2):
    z = np.asarray(logits, dtype=np.float32).astype(np.float64)
    rows = np.arange(len(z))
    wy, ly = w[rows, y], z[rows, y]
    out = np.full(len(z), np.inf)
    pos = s2 > 0
    with np.errstate(divide="ignore", invalid="ignore"):
        tau = ((ly[:, None] - z) * np.sqrt(s2)[:, None]) / (w - wy[:, None])
    tau = np.where(w > wy[:, None], tau, np.inf)
    out[pos] = tau[pos].min(axis=1)
    return out


def radius2(emb, anc):
    return T.exact_d2_table(emb, anc).max(axis=1)


def rho_from(t, r2, d):
    with np.errstate(divide="ignore", invalid="ignore"):
        v = (math.sqrt(d) * t) / np.sqrt(r2)
    return np.where((r2 > 0) & np.isfinite(t), v, np.inf)


def rho(logits, emb, anc, weight, parts=False):
    """rho [n] (and R2, t* with parts) for candidate logits [n, C], embeddings [n, Dp], anchors [C, Dp], head [C, D]."""
    y, _, w, s2 = head_terms(logits, weight)
    t = tstar(logits, y, w, s2)
    r2 = radius2(emb, anc)
    out = rho_from(t, r2, np.asarray(weight).shape[1])
    return (out, r2, t) if parts else out


# ---- the caps, the diversity step, the query ----------------------------------------------------------------------------
def cap_walk(rho_v, budget, alpha_step=ALPHA_STEP):
    """Positions {rho < kappa_j} of the first j with more than `budget` of them, else of the last j; one cap at a time."""
    rho_v = np.asarray(rho_v, dtype=np.float64)
    sel = np.zeros(0, dtype=np.int64)
    for j in range(1, math.ceil(1.0 / alpha_step) + 1):
        sel = np.flatnonzero(rho_v < j * alpha_step)
        if len(sel) > budget:
            break
    return sel


def nearest(xhat, labels, centres):
    """Per cluster id < K: the lowest row of the smallest exact_d2 to its centre among the rows labeled with it, -1 if none."""
    labels = np.asarray(labels, dtype=np.int64)
    d2 = P.exact_d2(xhat, centres[labels])
    out = np.full(len(centres), -1, dtype=np.int64)
    o = np.lexsort((np.arange(len(labels)), d2, labels))
    first = np.ones(len(o), dtype=bool)
    first[1:] = labels[o][1:] != labels[o][:-1]
    out[labels[o][first]] = o[first]
    return out


def diverse(emb_cand, budget, max_iter=MAX_ITER):
    """Positions into the candidates: all of them when they do not exceed the budget, else one per non-empty k-means
    cluster, drawing the seeding from NumPy."""
    n = len(emb_cand)
    if n <= budget:
        return np.arange(n, dtype=np.int64)
    xhat = T.normalize(emb_cand)
    first = int(np.random.choice(n))
    unif = np.random.random_sample(budget - 1)
    seeds = T.seed(xhat, first, unif, budget)
    labels, centres, _ = T.lloyd(xhat, xhat[seeds].copy(), max_iter)
    near = nearest(xhat, labels, centres)
    return near[near >= 0]


def query_positions(emb, logits, weight, labels_lab, is_lab, avail, budget, alpha_step=ALPHA_STEP, rho_v=None):
    """Positions in the pool that the query returns, in order.  `labels_lab` are the labeled rows' classes in position
    order; `rho_v` replaces the candidates' rho where a test supplies the device's."""
    budget = int(min(int(np.sum(avail)), budget))
    if budget <= 0:
        return np.zeros(0, dtype=np.int64)
    lab, cand = np.flatnonzero(is_lab), np.flatnonzero(avail)
    if not len(lab):
        raise ValueError("ALFAMixSampler needs labeled rows")
    emb, logits = np.asarray(emb, dtype=np.float32), np.asarray(logits, dtype=np.float32)
    if rho_v is None:
        anc = anchors(emb[lab], labels_lab, np.asarray(weight).shape[0])
        rho_v = rho(logits[cand], emb[cand], anc, weight)
    sel = cand[cap_walk(rho_v, budget, alpha_step)]
    picks = sel[diverse(emb[sel], budget)]
    return P.random_fill(picks, avail, budget)


# ---- the paper's mixing, literally ----------------------------------------------------------------------------------------
def literal_flips(emb, anc, weight, bias, eps):
    """Per row of emb [n, D]: does some anchor's mixed feature, at the closed-form alpha* for cap eps, change the head's
    fp64 prediction?  alpha* = eps |a - z| g / (|g| (a - z)) per coordinate with g = W^T (p - e_yhat) the loss gradient
    of the feature at the pseudo-label; the mixed feature (1 - alpha*) z + alpha* a goes through nn.Linear in fp64."""
    lin = torch.nn.Linear(weight.shape[1], weight.shape[0]).double()
    with torch.no_grad():
        lin.weight.copy_(torch.from_numpy(np.asarray(weight, dtype=np.float64)))
        lin.bias.copy_(torch.from_numpy(np.asarray(bias, dtype=np.float64)))
        z = torch.from_numpy(np.asarray(emb, dtype=np.float64))
        a = torch.from_numpy(np.asarray(anc, dtype=np.float64))
        logits = lin(z)
        yhat = logits.argmax(dim=1)
        p = torch.softmax(logits, dim=1)
        p[torch.arange(len(z)), yhat] -= 1.0
        g = p @ lin.weight                                               # [n, D]
        out = np.zeros(len(z), dtype=bool)
        for u in range(len(z)):
            diff = a - z[u]                                              # [C, D], no zero coordinate
            alpha = eps * diff.norm(dim=1, keepdim=True) * g[u] / (g[u].norm() * diff)
            mixed = (1 - alpha) * z[u] + alpha * a
            out[u] = bool((lin(mixed).argmax(dim=1) != yhat[u]).any())
        return out


# ---- K20's distance from `rho` ---------------------------------------------------------------------------------------------
ULPS = CO.ULPS


def rho_bound(logits, weight, rho_v):
    """Per row, a bound on |K20's rho - rho()| when both follow the same operation order and differ only in exp / log,
    each within ULPS ulp (DESIGN section 4): the error of p (from cal_oracle's bound on lse), carried through r, w = G r,
    s2 = r^T w and every tau_k near t* to first order, with the roundings of both chains on either side.  +inf for a row
    whose t* could change class because some w_k - w_yhat lies within its own error, or whose s2 lies within its own
    error (a prediction so confident that r_yhat = p_yhat - 1 cancels)."""
    z = np.asarray(logits, dtype=np.float32)
    g = gram(weight)
    y, r, w, s2 = head_terms(z, weight, g)
    t = tstar(z, y, w, s2)
    n, C = r.shape
    q = 2.0 * ULPS * U
    lse, lp = CO.log_softmax(z)
    dlp = 1.05 * (2 * q + 2 * (C + 2) * U + 2 * q * math.log(max(C, 2)) + 4 * U * np.abs(lse) + 4 * U * np.abs(lp).max(1))
    ep = 1.05 * (dlp + 2 * q)                                           # relative error of p
    p = np.abs(r)
    p[np.arange(n), y] = np.abs(r[np.arange(n), y] + 1.0)
    dr = ep[:, None] * p + 2 * U * np.abs(r)
    gam = 1.05 * 2 * (C + 2) * U
    ag = np.abs(g)
    dw = dr @ ag + gam * (np.abs(r) @ ag)
    ds2 = (np.abs(r) * dw + np.abs(w) * dr + dr * dw).sum(1) + gam * (np.abs(r) * np.abs(w)).sum(1)
    out = np.full(n, np.inf)
    rows = np.arange(n)
    wy, ly = w[rows, y], z.astype(np.float64)[rows, y]
    for u in range(n):
        if not np.isfinite(t[u]):                                       # exact when s2 is exactly 0 on both sides
            out[u] = 0.0 if s2[u] <= 0 and ds2[u] == 0 else np.inf
            continue
        if not ds2[u] < 0.5 * s2[u]:
            continue                                                    # s2 lost to cancellation in r_yhat = p - 1
        s = math.sqrt(s2[u])
        es = 1.05 * ds2[u] / (2 * s2[u] - 2 * ds2[u]) + 4 * U
        gap = w[u] - wy[u]
        dg = dw[u] + dw[u, y[u]] + 2 * U * np.abs(gap)
        near = gap > -dg
        near[y[u]] = False
        low = (ly[u] - z[u].astype(np.float64)) * s * (1 - es) / (np.maximum(gap, 0) + dg)
        sure = gap - dg > 0
        if (near & ~sure & (low <= t[u] * 1.01)).any():
            continue                                                    # a k of ambiguous sign may set t*
        k = near & sure & (low <= t[u] * 1.01)
        if not k.any():
            continue
        e = es + dg[k] / (gap[k] - dg[k]) + 8 * U
        out[u] = 1.1 * float(e.max()) * abs(rho_v[u]) + 8 * U * abs(rho_v[u])
    return out
