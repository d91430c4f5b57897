"""NumPy statement of BAITSampler's query (active_learning_b200/query_strategies/bait.py, kernels K24 / K25 / K26), written
from the algorithm of Ash, Goel, Krishnamurthy & Kakade, "Gone Fishing: Neural Active Learning with Fisher Embeddings"
(NeurIPS 2021).  Everything is fp64.

  pool       CoreSet's pool: n rows, L the labeled ones, the candidates the available ones, B the clamped budget;
  p_x        the softmax of the fp32 logits, lse = max + log sum exp(z - max) (cal_oracle's form);
  V_x        R_x (x) h_x^T, R_x = diag(sqrt p_x)(I - 1 p_x^T), coordinate (c, d) at c D + d, h_x the raw fp32 embedding;
             V_x^T V_x = (diag p - p p^T) (x) h h^T;
  F          (1/n) sum over the pool of V_x^T V_x;
  A          M0^-1, M0 = lamb I + sum_{l in L} V_l^T V_l / (|L| + B);
  forward    T = min(2B, #candidates) steps, Vt = sqrt(B / (|L| + B)) V: take the unpicked candidate of the largest
             tr((Vt A F A Vt^T)(I + Vt A Vt^T)^-1) (lowest position on ties), A <- A - A Vt^T (I + Vt A Vt^T)^-1 Vt A;
  backward   T - B steps: remove the first list entry of the largest tr((Vt A F A Vt^T)(-I + Vt A Vt^T)^-1),
             A <- A - A Vt^T (-I + Vt A Vt^T)^-1 Vt A;
  result     the list that remains, in forward-pick order.  No NumPy draw after the pool's shuffles.

`literal_select` transcribes that loop with V_x materialised and np.linalg.inv.  `select` is the factored, incremental
form the device follows: per row the C x C forms At_x[a, b] = h_x^T A_ab h_x and Gt_x[a, b] = h_x^T (A F A)_ab h_x (A_ab the
D x D block), so that Vt A Vt^T = s^2 R At R^T, kept through each rank-C update A <- A - U S U^T (U = A Vt_*^T) with
W_x[a, k] = h_x^T U_{a,k} and Z_x[a, k] = h_x^T (A F U)_{a,k}:
  At <- At - W S W^T,   Gt <- Gt - W S Z^T - Z S W^T + W S (U^T F U) S W^T.
The labeled rows are absorbed through the same update from A = I / lamb (At = |h|^2 / lamb I, Gt_ab = h^T F_ab h / lamb^2).
"""
import math

import numpy as np


def bait_lamb(lamb):
    """The sampler kwarg `lamb` as a float: ValueError unless it is finite and > 0."""
    try:
        v = float(lamb)
    except (TypeError, ValueError):
        raise ValueError(f"lamb={lamb!r} is not a number") from None
    if not (math.isfinite(v) and v > 0):
        raise ValueError(f"lamb must be finite and > 0, got {lamb!r}")
    return v


def bait_bytes(n, c, d):
    """Engine.bait_bytes: A, F and scratch at 8 dim^2 each, the two per-row forms at 8 n C^2 each."""
    dim = int(c) * int(d)
    return 3 * 8 * dim * dim + 2 * 8 * int(n) * int(c) * int(c)


def probs(logits):
    z = np.asarray(logits, dtype=np.float32).astype(np.float64)
    m = z.max(axis=1, keepdims=True)
    lse = m + np.log(np.exp(z - m).sum(axis=1, keepdims=True))
    return np.exp(z - lse)


def r_factor(p):
    """R = diag(sqrt p)(I - 1 p^T) for one row p [C]."""
    c = p.shape[0]
    return np.sqrt(p)[:, None] * (np.eye(c) - p[None, :])


def v_matrix(p, h):
    """V_x [C, C D]: row k is sqrt(p_k) (e_k - p) (x) h."""
    return np.kron(r_factor(p), np.asarray(h, dtype=np.float64)[None, :])


def fisher(logits, emb):
    """F [C D, C D] = (1/n) sum_x (diag p - p p^T) (x) h h^T."""
    p = probs(logits)
    h = np.asarray(emb, dtype=np.float32).astype(np.float64)
    n, c = p.shape
    d = h.shape[1]
    F = np.zeros((c * d, c * d))
    for a in range(c):
        for b in range(a, c):
            w = ((p[:, a] if a == b else 0.0) - p[:, a] * p[:, b]) / n
            blk = h.T @ (w[:, None] * h)
            if a == b:                        # exactly symmetric: the upper triangle mirrored, as the device does
                blk = np.triu(blk) + np.triu(blk, 1).T
            F[a * d:(a + 1) * d, b * d:(b + 1) * d] = blk
            F[b * d:(b + 1) * d, a * d:(a + 1) * d] = blk.T
    return F


def scales(n_lab, budget):
    """(1 / sqrt(|L| + B), sqrt(B / (|L| + B))): the labeled rows' and the candidates' scale of V."""
    return 1.0 / math.sqrt(n_lab + budget), math.sqrt(budget / (n_lab + budget))


def steps(n_cand, budget):
    return min(2 * int(budget), int(n_cand))


# ---- the literal transcription -----------------------------------------------------------------------------------------
def literal_select(logits, emb, is_lab, avail, budget, lamb=1.0):
    """The authors' loop in fp64 with V_x materialised: (positions in forward-pick order, forward scores, backward
    scores), the scores those of every step as {position: score}."""
    p = probs(logits)
    h = np.asarray(emb, dtype=np.float32).astype(np.float64)
    n, c = p.shape
    lab, cand = np.flatnonzero(is_lab), np.flatnonzero(avail)
    s_lab, s = scales(len(lab), budget)
    F = fisher(logits, emb)
    dim = F.shape[0]
    M0 = lamb * np.eye(dim)
    for l in lab:
        Vl = s_lab * v_matrix(p[l], h[l])
        M0 = M0 + Vl.T @ Vl
    A = np.linalg.inv(M0)
    X = np.stack([s * v_matrix(p[x], h[x]) for x in cand]) if len(cand) else np.zeros((0, c, dim))
    eye = np.eye(c)
    picked, fwd = [], []
    for _ in range(steps(len(cand), budget)):
        inner = np.linalg.inv(eye + X @ A @ X.transpose(0, 2, 1))
        score = np.trace(X @ A @ F @ A @ X.transpose(0, 2, 1) @ inner, axis1=1, axis2=2)
        free = np.ones(len(cand), dtype=bool)
        free[picked] = False
        fwd.append({int(cand[i]): float(score[i]) for i in np.flatnonzero(free)})
        i = int(np.flatnonzero(free)[np.argmax(score[free])])
        xt = X[i]
        A = A - A @ xt.T @ np.linalg.inv(eye + xt @ A @ xt.T) @ xt @ A
        picked.append(i)
    bwd = []
    for _ in range(len(picked) - int(budget)):
        xs = X[picked]
        inner = np.linalg.inv(-eye + xs @ A @ xs.transpose(0, 2, 1))
        r = np.trace(xs @ A @ F @ A @ xs.transpose(0, 2, 1) @ inner, axis1=1, axis2=2)
        bwd.append({int(cand[i]): float(v) for i, v in zip(picked, r)})
        j = int(np.argmax(r))
        xt = X[picked[j]]
        A = A - A @ xt.T @ np.linalg.inv(-eye + xt @ A @ xt.T) @ xt @ A
        del picked[j]
    return cand[np.asarray(picked, dtype=np.int64)], fwd, bwd


# ---- the factored, incremental form ------------------------------------------------------------------------------------
def sandwich(p, X):
    """R X R^T for rows p [m, C] and forms X [m, C, C]."""
    R = np.sqrt(p)[:, :, None] * (np.eye(p.shape[1])[None] - p[:, None, :])
    return R @ X @ R.transpose(0, 2, 1)


def initial_forms(emb, F, lamb):
    """A = I / lamb, At_x = |h_x|^2 / lamb I, Gt_x[a, b] = h_x^T F_ab h_x / lamb^2."""
    h = np.asarray(emb, dtype=np.float32).astype(np.float64)
    n, d = h.shape
    c = F.shape[0] // d
    A = np.eye(c * d) / lamb
    At = (h * h).sum(axis=1)[:, None, None] / lamb * np.eye(c)[None]
    Fb = F.reshape(c, d, c, d)
    Gt = np.einsum("xd,adbe,xe->xab", h, Fb, h) / (lamb * lamb)
    return A, At, Gt


def forms_scores(p, At, Gt, s, sigma):
    """tr((s^2 R Gt R^T)(sigma I + s^2 R At R^T)^-1) for rows p [m, C] and their forms."""
    c = p.shape[1]
    M = s * s * sandwich(p, At)
    G = s * s * sandwich(p, Gt)
    return np.trace(np.linalg.solve(sigma * np.eye(c)[None] + M, G), axis1=1, axis2=2)


def absorb(state, x, s, sigma):
    """The rank-C update of A and of every row's forms by row x at scale s: sigma = +1 adds s V_x, -1 removes it."""
    A, At, Gt, F, p, h = state["A"], state["At"], state["Gt"], state["F"], state["p"], state["h"]
    c = p.shape[1]
    d = h.shape[1]
    Vx = s * v_matrix(p[x], h[x])
    S = np.linalg.inv(sigma * np.eye(c) + Vx @ A @ Vx.T)
    U = A @ Vx.T
    FU = F @ U
    P = A @ FU
    Q = U.T @ FU
    W = np.einsum("xd,adk->xak", h, U.reshape(c, d, c))
    Z = np.einsum("xd,adk->xak", h, P.reshape(c, d, c))
    WS = W @ S
    state["At"] = At - WS @ W.transpose(0, 2, 1)
    ZSW = Z @ WS.transpose(0, 2, 1)
    state["Gt"] = Gt - ZSW.transpose(0, 2, 1) - ZSW + WS @ Q @ WS.transpose(0, 2, 1)
    state["A"] = A - U @ S @ U.T


def select(logits, emb, is_lab, avail, budget, lamb=1.0, F=None):
    """The incremental form: (positions in forward-pick order, forward scores, backward scores) as literal_select."""
    p = probs(logits)
    h = np.asarray(emb, dtype=np.float32).astype(np.float64)
    F = fisher(logits, emb) if F is None else F
    A, At, Gt = initial_forms(emb, F, lamb)
    st = {"A": A, "At": At, "Gt": Gt, "F": F, "p": p, "h": h}
    lab, cand = np.flatnonzero(is_lab), np.flatnonzero(avail)
    s_lab, s = scales(len(lab), budget)
    for l in lab:
        absorb(st, l, s_lab, 1.0)
    free = np.ones(len(cand), dtype=bool)
    picked, fwd = [], []
    for _ in range(steps(len(cand), budget)):
        rows = cand[free]
        score = forms_scores(p[rows], st["At"][rows], st["Gt"][rows], s, 1.0)
        fwd.append(dict(zip(rows.tolist(), score.tolist())))
        x = int(rows[int(np.argmax(score))])
        absorb(st, x, s, 1.0)
        free[np.searchsorted(cand, x)] = False
        picked.append(x)
    bwd = []
    for _ in range(len(picked) - int(budget)):
        rows = np.asarray(picked, dtype=np.int64)
        r = forms_scores(p[rows], st["At"][rows], st["Gt"][rows], s, -1.0)
        bwd.append(dict(zip(rows.tolist(), r.tolist())))
        j = int(np.argmax(r))
        absorb(st, picked[j], s, -1.0)
        del picked[j]
    return np.asarray(picked, dtype=np.int64), fwd, bwd


def separated(scores, rel=1e-8):
    """Whether the largest score of a step is tied exactly or ahead of the next distinct one by >= rel relative."""
    g = np.sort(np.array(list(scores.values())))[::-1]
    below = g[g < g[0]]
    return len(below) == 0 or g[0] - below[0] >= rel * abs(g[0])


def query_positions(logits, emb, is_lab, avail, budget, lamb=1.0):
    """Positions in the pool that the query returns, in forward-pick order."""
    budget = int(min(int(np.sum(avail)), budget))
    if budget <= 0:
        return np.zeros(0, dtype=np.int64)
    return select(logits, emb, is_lab, avail, budget, lamb)[0]
