"""CPU oracle for the per-round query path of zeyademam/active_learning.

TEST INFRASTRUCTURE ONLY.  This module is a CPU restatement (torch-CPU + NumPy, the same
third-party arithmetic the reference itself runs on) of the reference's acquisition
functions.  Only ``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` /
``--impl reference`` legs of ``bench.py`` may import it.  Nothing under
``active_learning_b200/`` imports it and the product path never falls back to it.

Parity status: PINNED.  Every function below is checked against outputs of the reference's
own code (imported in the build container from active_learning/src with a comet_ml stub) by
``tests/golden/make_golden.py``; the resulting vectors are committed under ``tests/golden/``
and ``tests/test_oracle_golden.py`` replays them.  The one exception is ``entropy`` scoring:
the reference has no EntropySampler (SURVEY.md finding 1), so that mode is *parity unpinned*
and its spec is defined here.  The MASE / BASE functions at the end (SURVEY.md section 8f rank 2)
are pinned the same way by ``tests/golden/make_golden_mase.py``, ``balancing_query`` by
``tests/golden/make_golden_balancing.py``.

All citations are relative to active_learning/src/query_strategies/.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

MODE_MARGIN = 0
MODE_LEAST_CONFIDENCE = 1
MODE_ENTROPY = 2

POOLING_H = 16      # badge_sampler.py:9
POOLING_AREA = 512  # badge_sampler.py:10


# --------------------------------------------------------------------------------------
# Softmax-uncertainty scores  (margin_sampler.py:29-43, confidence_sampler.py:27-45)
# --------------------------------------------------------------------------------------
def softmax_scores(logits: torch.Tensor, mode: int, batch_size: int = 128) -> torch.Tensor:
    """Per-row score, computed batch by batch exactly like the reference's loader loop.

    margin           : p(1) - p(2) of softmax(dim=1)            margin_sampler.py:33-35
    least confidence : p(1)                                     confidence_sampler.py:31-33
    entropy (NEW)    : -H = sum_c p_c * log p_c  (so "smallest first" == most uncertain first), with 0 log 0 = 0:
                       a masked class (logit -inf, p = 0) adds nothing.  A row with a NaN or +inf logit, or with every
                       logit -inf, still scores NaN.
    """
    logits = logits.detach().to(torch.float32).cpu()
    out = []
    for lo in range(0, logits.shape[0], batch_size):
        z = logits[lo:lo + batch_size]
        if mode == MODE_MARGIN:
            probs = torch.nn.Softmax(dim=1)(z)
            top, _ = probs.topk(dim=1, k=2, largest=True, sorted=True)
            out.append(top[:, 0] - top[:, 1])
        elif mode == MODE_LEAST_CONFIDENCE:
            probs = torch.nn.Softmax(dim=1)(z)
            top, _ = probs.topk(dim=1, k=1, largest=True, sorted=True)
            out.append(top[:, 0])
        elif mode == MODE_ENTROPY:
            logp = F.log_softmax(z, dim=1)
            p = logp.exp()
            out.append(torch.where(p == 0, torch.zeros(()), p * logp).sum(dim=1))
        else:
            raise ValueError(f"unknown mode {mode}")
    if not out:
        return torch.empty(0, dtype=torch.float32)
    return torch.cat(out, dim=0)


def select_smallest(scores: torch.Tensor, budget: int) -> np.ndarray:
    """Positions of the `budget` smallest scores, ascending, ties by lowest position.

    margin_sampler.py:41-42 uses torch.sort(descending=False) whose CPU kernel is stable in
    practice; the fixed tie-break of this build is "stable", stated explicitly here.
    """
    budget = int(min(len(scores), budget))
    order = torch.sort(scores, descending=False, stable=True).indices[:budget]
    return order.numpy().astype(np.int64)


def uncertainty_query(logits: torch.Tensor, idxs_for_query: np.ndarray, budget, mode: int,
                      batch_size: int = 128):
    """Tail of MarginSampler.query / ConfidenceSampler.query (line 41 of the latter removed,
    SURVEY.md finding 2): scores over the pool in loader order -> first `budget` by
    ascending score -> global indices."""
    scores = softmax_scores(logits, mode, batch_size)
    budget = int(min(len(idxs_for_query), budget))
    pos = select_smallest(scores, budget)
    return np.asarray(idxs_for_query)[pos].tolist(), budget


# --------------------------------------------------------------------------------------
# BADGE gradient embeddings  (badge_sampler.py:22-48)
# --------------------------------------------------------------------------------------
def gradient_embeddings(logits: torch.Tensor, emb: torch.Tensor, batch_size: int,
                        use_adaptive_pool: bool = False) -> torch.Tensor:
    """Materialised gradient embedding, batch by batch, through autograd like the reference:
    CE(mean) against the arg-max pseudo label (badge_sampler.py:33-37), outer product with
    the penultimate embedding (:40), optional 2-D adaptive average pool (:41-44)."""
    logits = logits.detach().to(torch.float32).cpu()
    emb = emb.detach().to(torch.float32).cpu()
    chunks = []
    for lo in range(0, logits.shape[0], batch_size):
        z = logits[lo:lo + batch_size].clone()
        h = emb[lo:lo + batch_size]
        pseudo = z.max(dim=1).indices
        z.requires_grad_(True)
        loss = torch.nn.CrossEntropyLoss()(z, pseudo)
        g = torch.autograd.grad(loss, z)[0]
        with torch.no_grad():
            ge = g[:, :, None] * h[:, None, :]
            if use_adaptive_pool:
                ph = min(POOLING_H, ge.size(1))
                pw = int(float(POOLING_AREA) / ph)
                ge = F.adaptive_avg_pool2d(ge, (ph, pw))
            chunks.append(ge.reshape(ge.size(0), -1))
    return torch.cat(chunks, dim=0)


def badge_factors(logits: torch.Tensor, batch_size: int) -> torch.Tensor:
    """Closed form of the logits-gradient above: a_i = (softmax(z_i) - onehot(argmax z_i)) / bs_i
    where bs_i is the size of the loader batch row i falls in (SURVEY.md finding 5).  The
    gradient embedding is the rank-1 matrix a_i (x) h_i (finding 6)."""
    logits = logits.detach().to(torch.float32).cpu()
    n = logits.shape[0]
    p = torch.softmax(logits, dim=1)
    onehot = F.one_hot(logits.max(dim=1).indices, logits.shape[1]).to(torch.float32)
    bs = torch.full((n,), float(batch_size))
    tail = n % batch_size
    if tail:
        bs[n - tail:] = float(tail)
    return (p - onehot) / bs[:, None]


def adaptive_pool_bins(n_in: int, n_out: int):
    """Window [start, end) of every adaptive_avg_pool output bin (ATen's start=floor(i*in/out),
    end=ceil((i+1)*in/out))."""
    return [((i * n_in) // n_out, -((-(i + 1) * n_in) // n_out)) for i in range(n_out)]


def pooled_factors(a: torch.Tensor, h: torch.Tensor):
    """1-D pooled factors whose outer product equals the reference's 2-D pooled embedding
    (SURVEY.md finding 6: pooling preserves rank-1)."""
    ph = min(POOLING_H, a.shape[1])
    pw = int(float(POOLING_AREA) / ph)
    pa = F.adaptive_avg_pool1d(a[:, None, :], ph)[:, 0, :]
    phh = F.adaptive_avg_pool1d(h[:, None, :], pw)[:, 0, :]
    return pa, phh


# --------------------------------------------------------------------------------------
# CoreSet / k-means++  (coreset_sampler.py:59-105)
# --------------------------------------------------------------------------------------
def pairwise_l2_dist(features: torch.Tensor) -> torch.Tensor:
    """Dense squared-L2 matrix, n_i + n_j - 2<e_i,e_j>  (coreset_sampler.py:59-64)."""
    features = features.to(torch.float32).cpu()
    n = features.shape[0]
    sq = features.square().sum(dim=1, keepdims=True).repeat((1, n))
    gram = torch.mm(features, features.T)
    return sq + sq.T - 2 * gram


def coreset(dist: torch.Tensor, labeled_indicator: np.ndarray, query_count: int,
            randomize: bool = False):
    """Greedy k-center (randomize=False, coreset_sampler.py:94) or D^2 sampling
    (randomize=True, :80-92) over a dense distance matrix.  Consumes the *global* NumPy RNG
    in the reference's order: one np.random.choice per step."""
    lab = np.array(labeled_indicator, dtype=bool, copy=True)
    picks = []
    for _ in range(int(query_count)):
        if lab.sum() > 0:
            mind = dist[:, lab].min(dim=1).values
            if randomize:
                mind = mind.cpu().numpy()
                while True:
                    prob = np.clip(mind, 0, None)
                    prob[lab] = 0.0
                    prob = prob / np.sum(prob)
                    if not np.isnan(prob.sum()):
                        break
                    mind += 0.00001
                q = np.random.choice(len(prob), p=prob)
            else:
                q = mind.max(dim=0).indices.item()
        else:
            if randomize:
                q = np.random.choice(len(lab))
            else:
                q = dist.max(dim=1).values.min(dim=0).indices.item()
        picks.append(int(q))
        lab[q] = True
    return picks


def np_pairwise_sum_f32(a: np.ndarray) -> np.float32:
    """Bit-exact restatement of NumPy's float32 add-reduce over a contiguous 1-D array
    (numpy/_core/src/umath/loops_utils.h.src `pairwise_sum`, NumPy 2.3.5; the structure is
    verified against np.sum in tests/test_oracle_golden.py).  Blocks of <=128 use 8 strided
    accumulators; larger inputs split at n/2 rounded down to a multiple of 8."""
    a = np.asarray(a, dtype=np.float32)
    n = a.shape[0]
    f = np.float32
    if n < 8:
        r = f(0.0)
        for x in a:
            r = f(r + x)
        return r
    if n <= 128:
        r = [f(a[j]) for j in range(8)]
        stop = n - (n % 8)
        for i in range(8, stop, 8):
            for j in range(8):
                r[j] = f(r[j] + a[i + j])
        res = f(f(f(r[0] + r[1]) + f(r[2] + r[3])) + f(f(r[4] + r[5]) + f(r[6] + r[7])))
        for i in range(stop, n):
            res = f(res + a[i])
        return res
    half = n // 2
    half -= half % 8
    return f(np_pairwise_sum_f32(a[:half]) + np_pairwise_sum_f32(a[half:]))


def pairwise_leaves(n: int):
    """Leaf segments [(start, length)] of the pairwise-sum recursion tree for length n, in
    left-to-right order (used to cross-check the host-side schedule the CUDA path uploads)."""
    out = []

    def rec(lo, m):
        if m <= 128:
            out.append((lo, m))
            return
        half = m // 2
        half -= half % 8
        rec(lo, half)
        rec(lo + half, m - half)

    rec(0, int(n))
    return out


def choice_from_uniform(prob32: np.ndarray, u: float) -> int:
    """np.random.choice(len(p), p=p) given the single uniform it draws (numpy/random/mtrand.pyx
    `choice`: cdf = cumsum(p as float64); cdf /= cdf[-1]; searchsorted(u, side='right'))."""
    cdf = np.asarray(prob32, dtype=np.float64).cumsum()
    cdf /= cdf[-1]
    return int(cdf.searchsorted(u, side="right"))


def d2_probabilities(mind32: np.ndarray, labeled: np.ndarray) -> np.ndarray:
    """The float32 `p` one randomize=True step of `coreset` hands to np.random.choice, including the
    `sum == 0 -> NaN -> += 1e-5` retry (coreset_sampler.py:82-90)."""
    mind = np.array(mind32, dtype=np.float32, copy=True)
    while True:
        prob = np.clip(mind, 0, None)
        prob[labeled] = 0.0
        prob = prob / np.sum(prob)
        if not np.isnan(prob.sum()):
            return prob
        mind += 0.00001


def d2_cdf(prob32: np.ndarray) -> np.ndarray:
    """np.random.choice's normalised fp64 cdf of `prob32` (see `choice_from_uniform`)."""
    cdf = np.asarray(prob32, dtype=np.float64).cumsum()
    cdf /= cdf[-1]
    return cdf


def d2_sampling_step(mind32: np.ndarray, labeled: np.ndarray, u: float) -> int:
    """One randomize=True step of `coreset` with the uniform made explicit
    (coreset_sampler.py:82-92)."""
    return choice_from_uniform(d2_probabilities(mind32, labeled), u)


def coreset_streaming(feat: torch.Tensor, labeled_indicator: np.ndarray, query_count: int,
                      randomize: bool = False, uniforms=None, factors: torch.Tensor = None, certificate=None):
    """Same picks as `coreset(pairwise_l2_dist(feat), ...)` but O(N) memory: running min of
    fl(fl(n_i+n_q) - 2*dot) against each new centre (min is exact, SURVEY.md finding 4).
    Used for the parity cases too large for a dense N x N matrix.  With `uniforms` given the
    RNG is not touched; `uniforms` is either an array (u of step t = uniforms[t]) or a callable
    u = uniforms(t, cdf) that sees np.random.choice's normalised cdf of step t (`d2_cdf`), so a test can
    place u exactly on, or just beside, a cdf breakpoint.

    factors: BADGE's second factor a[n, C].  The row of the reference's matrix is the gradient embedding
    g_i = a_i (x) h_i (badge_sampler.py:40) with h = feat; it is rank-1 (SURVEY.md finding 6), so
    <g_i, g_q> = <a_i, a_q> <h_i, h_q> and |g_i|^2 = |a_i|^2 |h_i|^2 and the 2048*1000-d rows are never formed
    (at C = 1000, D = 2048 they cannot be: 8 MB per row).  On exact-arithmetic (small integer) fixtures this is
    bit-identical to the materialised path (tests/test_oracle_golden.py pins the two against each other).

    certificate: optional list; per step one float is appended -- arg-max: the gap between the largest and the
    second-largest candidate min-distance (how far the pick is from a tie); D^2 draw: the distance of u from the
    nearest cdf breakpoint.  A GPU path whose distances differ in the last bits can only diverge where it is tiny."""
    feat = feat.to(torch.float32).cpu()
    lab = np.array(labeled_indicator, dtype=bool, copy=True)
    n = feat.shape[0]
    sq = feat.square().sum(dim=1)
    fa = None
    if factors is not None:
        fa = factors.to(torch.float32).cpu()
        sq = sq * fa.square().sum(dim=1)

    def dots(rows):                       # <g_i, g_j> for j in rows
        dp = feat @ feat[rows].T if rows.dim() else feat @ feat[rows]
        if fa is not None:
            dp = dp * (fa @ fa[rows].T if rows.dim() else fa @ fa[rows])
        return dp

    mind = torch.full((n,), float("inf"))
    lab_idx = np.flatnonzero(lab)
    for lo in range(0, len(lab_idx), 4096):
        j = torch.from_numpy(lab_idx[lo:lo + 4096])
        d = (sq[:, None] + sq[j][None, :]) - 2 * dots(j)
        mind = torch.minimum(mind, d.min(dim=1).values)
    picks = []
    for t in range(int(query_count)):
        if lab.sum() == 0:
            raise ValueError("coreset_streaming needs at least one labeled row")
        if randomize:
            cdf = d2_cdf(d2_probabilities(mind.numpy(), lab))
            if callable(uniforms):
                u = float(uniforms(t, cdf))
            else:
                u = float(uniforms[t]) if uniforms is not None else float(np.random.random_sample())
            q = int(cdf.searchsorted(u, side="right"))
            if certificate is not None:
                near = [abs(cdf[q] - u)] + ([abs(u - cdf[q - 1])] if q > 0 else [])
                certificate.append(float(min(near)))
        else:
            q = int(mind.max(dim=0).indices.item())
            if certificate is not None:
                top2 = torch.topk(mind, 2).values
                certificate.append(float(top2[0] - top2[1]))
        picks.append(q)
        lab[q] = True
        d = (sq + sq[q]) - 2 * dots(torch.tensor(q))
        mind = torch.minimum(mind, d)
    return picks


# --------------------------------------------------------------------------------------
# Host bookkeeping  (strategy.py:126-163, coreset_sampler.py:21-41,
#                    partitioned_coreset_sampler.py:36-47)
# --------------------------------------------------------------------------------------
def available_query_idxs(idxs_lb: np.ndarray, eval_idxs, shuffle: bool = True) -> np.ndarray:
    cand = np.where(idxs_lb == False)[0]  # noqa: E712  (strategy.py:141)
    if shuffle:
        cand = np.random.permutation(cand)
    ev = set(int(e) for e in eval_idxs)
    return np.array([x for x in cand if x not in ev])


def already_labeled_idxs(idxs_lb: np.ndarray, shuffle: bool = False) -> np.ndarray:
    lab = np.argwhere(idxs_lb).squeeze()
    if shuffle:
        lab = np.random.permutation(lab)
    return lab


def idxs_for_coreset(idxs_lb, eval_idxs, subset_labeled, subset_unlabeled):
    """coreset_sampler.py:21-41: returns (sorted union, labeled list, unlabeled list)."""
    unl = available_query_idxs(idxs_lb, eval_idxs, shuffle=True)
    lab = already_labeled_idxs(idxs_lb, shuffle=True)
    if subset_labeled is not None:
        k = min(subset_labeled, len(lab))
        lab = lab[:k]
    if subset_unlabeled is not None:
        cap = (subset_labeled + subset_unlabeled - k) if subset_labeled is not None \
            else subset_unlabeled
        unl = unl[:min(cap, len(unl))]
    return sorted(unl.tolist() + lab.tolist()), lab.tolist(), unl.tolist()


def partition_idxs(input_idxs, partitions: int):
    """partitioned_coreset_sampler.py:36-47."""
    idxs = np.array(input_idxs)
    np.random.shuffle(idxs)
    out, cum = [], 0
    for i in range(partitions):
        m = int(len(input_idxs) / partitions) + int(i < len(input_idxs) % partitions)
        out.append(idxs[cum:cum + m])
        cum += m
    return out


# --------------------------------------------------------------------------------------
# MASE / BASE  (mase_sampler.py:29-102, base_sampler.py:12-44)
# --------------------------------------------------------------------------------------
def mase_margins(emb: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, batch_size: int = 128):
    """Distance of every embedding to each pairwise decision boundary of the linear head, restated from
    mase_sampler.py:52-80 batch by batch with the reference's own broadcast arithmetic:
        pred = argmax(linear(h));  wd = w_pred - w_c;  lam = 2 (h.wd + b_pred - b_c) / |wd|^2;
        radius_c = | -wd * lam / 2 |;  NaN (c == pred, duplicated class rows) -> inf;  min over c.
    Returns (min_margins [N], per_class_margins [N, C], pred [N])."""
    emb = emb.detach().to(torch.float32).cpu()
    weight = weight.detach().to(torch.float32).cpu()
    bias = bias.detach().to(torch.float32).cpu()
    mins, radii, preds = [], [], []
    for lo in range(0, emb.shape[0], batch_size):
        h = emb[lo:lo + batch_size]
        logits = F.linear(h, weight, bias)
        pred = logits.max(dim=1).indices                                   # :57
        wd = weight[pred, :][:, None, :] - weight[None, :]                 # :60-62  (B, C, M)
        bd = bias[pred, None] - bias[None, :]                              # :65
        lam_num = 2 * ((h[:, None, :] * wd).sum(dim=2) + bd)               # :68
        lam_den = (wd ** 2).sum(dim=2)                                     # :71
        lam = lam_num / lam_den
        eps = -wd * lam[:, :, None] / 2                                    # :74
        radius = torch.linalg.norm(eps, dim=2)                             # :76
        radius = torch.where(torch.isnan(radius), torch.tensor(float("inf")), radius)   # :77
        m, _ = radius.min(dim=1)                                           # :79
        mins.append(m)
        radii.append(radius)
        preds.append(pred)
    if not mins:
        c = weight.shape[0]
        return torch.empty(0), torch.empty(0, c), torch.empty(0, dtype=torch.int64)
    return torch.cat(mins), torch.cat(radii), torch.cat(preds)


def mase_margins_closed_form(logits: torch.Tensor, weight: torch.Tensor):
    """The same quantity with the algebra carried out: h.wd + b_pred - b_c is the logit gap z_pred - z_c, and
    | -wd * lam / 2 | = |z_pred - z_c| / |w_pred - w_c|.  Equal to `mase_margins` up to fp32 rounding of the two
    evaluation orders (checked in tests/test_oracle_golden_mase.py); this is the form a streaming kernel
    evaluates, and the one usable at sizes where the (B, C, M) broadcast of the reference does not fit."""
    z = logits.detach().to(torch.float32).cpu()
    w = weight.detach().to(torch.float32).cpu()
    pred = z.max(dim=1).indices
    den = ((w[:, None, :] - w[None, :, :]) ** 2).sum(dim=2)                # [C, C]
    gap = (z.gather(1, pred[:, None]) - z).abs()
    radius = gap / den.sqrt()[pred]
    radius = torch.where(torch.isnan(radius), torch.tensor(float("inf")), radius)
    radius[torch.arange(z.shape[0]), pred] = float("inf")
    return radius.min(dim=1).values, radius, pred


def mase_query(min_margins: torch.Tensor, idxs_for_query: np.ndarray, budget):
    """mase_sampler.py:23-27 under the fixed tie-break (stable)."""
    budget = int(min(len(idxs_for_query), budget))
    pos = select_smallest(min_margins, budget)
    return np.asarray(idxs_for_query)[pos].tolist(), budget


def base_select(min_margins: torch.Tensor, per_class_margins: torch.Tensor, pred: torch.Tensor,
                budget: int, num_classes: int):
    """base_sampler.py:22-38: class by class, the `budget // C (+1)` rows closest to that class's boundary --
    rows predicted as c compete with their overall minimum margin, the others with their distance to class c;
    rows already taken are pushed to inf.  Sorts are stable (fixed tie-break).  Returns pool positions in
    pick order; raises like the reference's assert (:40) if a row would be taken twice."""
    mm = min_margins.detach().to(torch.float32).cpu()
    pc = per_class_margins.detach().to(torch.float32).cpu()
    pred = pred.detach().cpu()
    picked = []
    for c in range(num_classes):
        count = int(budget / num_classes) + int(c < budget % num_classes)
        if count == 0:
            continue
        key = torch.where(pred == c, mm, pc[:, c])
        if picked:
            key[picked] = float("inf")
        picked += select_smallest(key, count).tolist()
    assert len(picked) == len(set(picked))
    return np.asarray(picked, dtype=np.int64)


# --------------------------------------------------------------------------------------
# BalancingSampler  (balancing_sampler.py:26-134)
# --------------------------------------------------------------------------------------
def balancing_query(embeddings: torch.Tensor, ys: torch.Tensor, idxs_for_query: np.ndarray, idxs_labeled: np.ndarray,
                    budget, num_classes: int, diag: dict | None = None):
    """balancing_sampler.py:58-134, one pick per step: if the labeled class histogram is imbalanced relative to the
    remaining budget (:81-82), take the available row that minimises
        d2(row, centre of the rarest class) / max_{majority classes} d2(row, centre)      (:95-120, first index on ties),
    with class centres = mean labeled embedding (count + 1e-5 in the denominator, :86-88) and numerator 1 when the
    rarest class has no labeled row (:104-107); otherwise one `np.random.choice` over the available rows (:124).
    `idxs_for_query` / `idxs_labeled` are boolean masks over the pool and are updated like the reference's (:127-128).
    `diag["min_rel_gap"]` receives the smallest relative gap between the two smallest ratios of any balancing step."""
    embeddings = embeddings.detach().to(torch.float32).cpu()
    ys = ys.detach().cpu()
    idxs_for_query = np.array(idxs_for_query, dtype=bool)
    idxs_labeled = np.array(idxs_labeled, dtype=bool)
    budget = int(min(idxs_for_query.sum(), budget))
    picks, gap, n_bal = [], float("inf"), 0
    for query_count in range(budget):
        ys_labeled = ys[idxs_labeled]
        count = (ys_labeled[None, :] == torch.arange(num_classes)[:, None]).sum(dim=1)             # :66-67
        labeled_count = idxs_labeled.sum()
        mean_count = count.float().mean()
        maj = count > mean_count                                                                    # :71
        maj_avg = count[maj].sum() / maj.sum()
        minor = count <= mean_count
        minor_avg = count[minor].sum() / minor.sum()
        if budget - query_count <= minor.sum() * (maj_avg - minor_avg):                             # :81-82
            emb_l = embeddings[idxs_labeled]
            avg = torch.zeros(num_classes, labeled_count)                                           # :86-88
            avg[ys_labeled, torch.arange(len(ys_labeled))] = 1
            avg = avg / (avg.sum(dim=1, keepdims=True) + 1e-5)
            centres = avg @ emb_l
            c_major = centres[maj]
            rare_count, rare = count.min(dim=0)
            c_rare = centres[rare][None, :]
            emb_u = embeddings[idxs_for_query]
            a2 = emb_u.square().sum(dim=1, keepdims=True)
            d_rare = a2 + c_rare.square().sum(dim=1, keepdims=True).T - 2 * (emb_u @ c_rare.T)      # :98-101
            if rare_count == 0:
                d_rare = torch.ones_like(d_rare)
            d_major = a2 + c_major.square().sum(dim=1, keepdims=True).T - 2 * (emb_u @ c_major.T)   # :109-112
            ratio = (d_rare / d_major.max(dim=1, keepdims=True).values).squeeze()                   # :114-117
            q_in = ratio.min(dim=0).indices
            query_idx = np.where(idxs_for_query)[0][q_in]
            if ratio.numel() > 1:
                two = torch.topk(ratio.double().reshape(-1), 2, largest=False).values
                gap = min(gap, float((two[1] - two[0]) / two[1].abs().clamp_min(1e-30)))
            n_bal += 1
        else:
            query_idx = np.random.choice(np.where(idxs_for_query.squeeze())[0])                     # :124
        idxs_for_query[query_idx] = False
        idxs_labeled[query_idx] = True
        picks.append(int(query_idx))
    if diag is not None:
        diag["min_rel_gap"], diag["balancing_steps"] = gap, n_bal
    return picks, len(picks)
