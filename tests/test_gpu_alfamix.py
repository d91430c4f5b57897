"""ALFAMixSampler on the H100 (K20, K21, K15 / K16 past 8 192 clusters, and the query around them) against the NumPy
statement in alfamix_oracle.py: R^2 and K21 bit for bit, rho within the bound that CUDA's exp / log allow, the picks and
the NumPy state equal to the oracle's."""
import numpy as np
import pytest
import torch

import alfamix_oracle as AO
import probcover_oracle as P
import typiclust_oracle as T
from helpers import HeadNet, LabeledIndexDataset, make_strategy
from test_gpu_typiclust import _clustered, _exact_rows

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from active_learning_b200.engine import Engine
    return Engine()


def _check_rho(eng, logits, emb, anc, w):
    rho, r2, t = eng.alfamix_rho(*(torch.from_numpy(v).cuda() for v in (logits, emb, anc, w)), want_parts=True)
    rho, r2, t = rho.cpu().numpy(), r2.cpu().numpy(), t.cpu().numpy()
    want, want_r2, want_t = AO.rho(logits, emb, anc, w, parts=True)
    assert (r2.view(np.uint64) == want_r2.view(np.uint64)).all()
    bound = AO.rho_bound(logits, w, want)
    ok = np.isfinite(bound)
    assert ok.mean() > 0.95
    assert (np.isinf(rho[ok]) == np.isinf(want[ok])).all()
    fin = ok & np.isfinite(want)
    err = np.abs(rho[fin] - want[fin])
    assert (err <= bound[fin]).all(), float((err / np.maximum(bound[fin], 1e-300)).max())
    tb = bound[fin] / np.maximum(want[fin], 1e-300) * want_t[fin]       # the same relative bound for t*
    assert (np.abs(t[fin] - want_t[fin]) <= tb * 1.0001 + 1e-300).all()
    return rho


@pytest.mark.parametrize("n,c,d,dp", [(3000, 2, 12, 12), (3000, 10, 36, 36), (2000, 100, 510, 512), (600, 1000, 64, 64)])
def test_rho_within_the_bound_and_r2_bit_for_bit(eng, n, c, d, dp):
    rng = np.random.default_rng(n + c + d)
    w = (rng.normal(size=(c, d)) * 0.3).astype(np.float32)
    emb = np.zeros((n, dp), dtype=np.float32)
    emb[:, :d] = _clustered(n, d, 20, d, noise=0.5) * 10.0 ** rng.uniform(-1, 1, size=(n, 1)).astype(np.float32)
    logits = (rng.normal(size=(n, c)) * 3).astype(np.float32)
    logits[:50, 0] = np.clip(logits[:50, 0] * 20, -80, 80)              # large logits
    logits[5] = 0.0                                                     # a flat row
    anc = np.zeros((c, dp), dtype=np.float32)
    anc[:, :d] = (rng.normal(size=(c, d))).astype(np.float32)
    emb[7] = anc[0]                                                     # a row on an anchor
    rho = _check_rho(eng, logits, emb, anc, w)
    assert np.isfinite(rho).mean() > 0.9


def test_kmeans_nearest_bit_for_bit(eng):
    rng = np.random.default_rng(3)
    for n, d, k in ((5000, 36, 300), (4000, 520, 700), (300, 4, 40)):
        xhat = T.normalize(_clustered(n, d, max(2, k // 3), d))
        xhat[n // 2:n // 2 + 20] = xhat[n // 3]                          # duplicates: ties go to the lowest row
        centres = xhat[rng.choice(n, k, replace=False)].copy()
        labels = T.assign(xhat, centres)
        labels[labels == 1] = 2                                         # an empty cluster
        labels[:7] = -1                                                 # rows outside [0, K) are skipped
        got = eng.kmeans_nearest(torch.from_numpy(xhat).cuda(), torch.from_numpy(labels.astype(np.int32)).cuda(),
                                 torch.from_numpy(centres).cuda())
        want = AO.nearest(xhat[7:], labels[7:], centres)
        want = np.where(want >= 0, want + 7, -1)
        assert got.tolist() == want.tolist() and got[1] == -1


def test_kmeans_past_the_old_cluster_cap(eng):
    n, d, k = 12000, 36, 10000
    rng = np.random.default_rng(9)
    xhat = T.normalize(_clustered(n, d, 400, 9))
    first, unif = int(rng.integers(n)), rng.random(k - 1)
    labels, centres, it, seeds = eng.kmeans(torch.from_numpy(xhat).cuda(), first, unif, k)
    want_l, want_c, want_it = T.lloyd(xhat, xhat[seeds].copy())
    assert len(set(seeds.tolist())) == k and it == want_it
    assert labels.cpu().numpy().tolist() == want_l.tolist()
    assert (centres.cpu().numpy().view(np.uint32) == want_c.view(np.uint32)).all()


def _e2e(eng, n, d, c, n_lab, seed):
    rng = np.random.default_rng(seed)
    emb = _exact_rows(rng, n, d)
    w = rng.integers(-2, 3, size=(c, d)).astype(np.float32)
    bias = rng.integers(-2, 3, size=c).astype(np.float32)
    ys = rng.integers(0, c, size=n)
    net = HeadNet(torch.from_numpy(emb), torch.from_numpy(w), torch.from_numpy(bias))
    ev = rng.choice(n, 50, replace=False)
    lab = rng.choice(np.setdiff1d(np.arange(n), ev), n_lab, replace=False)
    s = make_strategy("ALFAMixSampler", None, None, ev, lab, 4096, engine=eng, net=net,
                      dataset=LabeledIndexDataset(ys, c))
    return s, emb, w, ys


@pytest.mark.parametrize("n,d,c,budgets", [(50000, 512, 10, (1000, 1000)), (20000, 512, 100, (9000, 9000))])
def test_query_equals_the_oracle_over_two_rounds(eng, n, d, c, budgets):
    s, emb, w, ys = _e2e(eng, n, d, c, 500, n + c)
    for rnd, budget in enumerate(budgets):
        np.random.seed(100 + rnd)
        got, k = s.query(budget)
        after = np.random.get_state()
        np.random.seed(100 + rnd)
        union = np.asarray(s.get_idxs_for_coreset(), dtype=np.int64)
        is_lab = s.already_labeled_idxs(boolean=True)[union]
        avail = s.available_query_idxs(boolean=True)[union]
        with torch.no_grad():
            logits = s.net.linear(torch.from_numpy(emb[union]).cuda()).cpu().numpy()
        e, lab_y = emb[union], ys[union][is_lab]
        cand = np.flatnonzero(avail)
        want_rho = AO.rho(logits[cand], e[cand], AO.anchors(e[is_lab], lab_y, c), w)
        kappa = np.arange(1, 33) * AO.ALPHA_STEP
        fin = np.isfinite(want_rho)
        assert (np.abs(want_rho[fin, None] - kappa) > 1e-9 * kappa).all()    # no rho within rounding of a cap
        want = union[AO.query_positions(e, logits, w, lab_y, is_lab, avail, budget, rho_v=want_rho)].tolist()
        assert got == want and k == budget
        assert (np.random.get_state()[1] == after[1]).all() and np.random.get_state()[2] == after[2]
        s.update(got, k)
        s.round += 1
        with torch.no_grad():
            s.net.linear.bias.add_(1.0)


def test_imagenet_lt_shape(eng):
    n, d, c, budget = 115846, 2048, 1000, 10000
    rng = np.random.default_rng(17)
    g = torch.Generator().manual_seed(17)
    cen = torch.randn(300, d, generator=g)
    emb = cen[torch.randint(0, 300, (n,), generator=g)] + 0.6 * torch.randn(n, d, generator=g)
    w = torch.randn(c, d, generator=g) * 0.05
    ys = rng.integers(0, c, size=n)
    net = HeadNet(emb, w, torch.zeros(c))
    lab = rng.choice(n, n // 10, replace=False)
    s = make_strategy("ALFAMixSampler", None, None, [], lab, 4096, engine=eng, net=net, dataset=LabeledIndexDataset(ys, c))
    np.random.seed(3)
    got, k = s.query(budget)
    after = np.random.get_state()
    # the query replayed on the engine, every piece of it checked against its own statement
    np.random.seed(3)
    union = np.asarray(s.get_idxs_for_coreset(), dtype=np.int64)
    is_lab = s.already_labeled_idxs(boolean=True)[union]
    avail = s.available_query_idxs(boolean=True)[union]
    cand = np.flatnonzero(avail)
    e = emb.cuda()[torch.from_numpy(union).cuda()]
    with torch.no_grad():                                               # the forward's batches: the same GEMM shapes
        logits = torch.cat([s.net.linear(e[lo:lo + 4096]) for lo in range(0, n, 4096)])
    anc = s._anchors(e[torch.from_numpy(np.flatnonzero(is_lab)).cuda()], ys[union][is_lab], c)
    ct = torch.from_numpy(cand).cuda()
    rho, r2, _ = eng.alfamix_rho(logits[ct], e[ct], anc, net.linear.weight.detach().cuda(), want_parts=True)
    rho, r2 = rho.cpu().numpy(), r2.cpu().numpy()
    rows = np.sort(rng.choice(len(cand), 300, replace=False))
    lg, eh, ah, wh = logits[ct].cpu().numpy()[rows], e[ct].cpu().numpy()[rows], anc.cpu().numpy(), w.numpy()
    want, want_r2, _ = AO.rho(lg, eh, ah, wh, parts=True)
    assert (r2[rows].view(np.uint64) == want_r2.view(np.uint64)).all()
    bound = AO.rho_bound(lg, wh, want)
    ok = np.isfinite(bound) & np.isfinite(want)
    assert ok.mean() > 0.95 and (np.abs(rho[rows][ok] - want[ok]) <= bound[ok]).all()
    sel = cand[AO.cap_walk(rho, budget)]
    assert len(sel) > budget
    xhat = eng.normalize(e[torch.from_numpy(sel).cuda()])
    first = int(np.random.choice(len(sel)))
    unif = np.random.random_sample(budget - 1)
    labels, centres, _, _ = eng.kmeans(xhat, first, unif, budget)
    near = eng.kmeans_nearest(xhat, labels, centres)
    picks = sel[near[near >= 0]]
    picks = P.random_fill(picks, avail, budget)
    assert got == union[picks].tolist() and k == budget
    assert (np.random.get_state()[1] == after[1]).all() and np.random.get_state()[2] == after[2]
    # K21's choice is the exact fp64 argmin over its cluster's members
    lab_h, xh, ch = labels.cpu().numpy(), xhat.cpu().numpy(), centres.cpu().numpy()
    for cl in rng.choice(np.flatnonzero(near >= 0), 12, replace=False):
        mem = np.flatnonzero(lab_h == cl)
        d2 = P.exact_d2(xh[mem], np.repeat(ch[cl:cl + 1], len(mem), axis=0))
        assert near[cl] == mem[np.lexsort((mem, d2))[0]]
    assert len(set(got)) == budget and not np.isin(got, lab).any()


def test_errors_are_clean_and_leave_the_context_usable(eng):
    from active_learning_b200._lib import AlqError
    rng = np.random.default_rng(1)
    logits = torch.randn(200, 10, device="cuda")
    emb = torch.randn(200, 16, device="cuda")
    anc = torch.randn(10, 16, device="cuda")
    w = torch.randn(10, 16, device="cuda")
    for which in range(4):
        args = [t.clone() for t in (logits, emb, anc, w)]
        args[which][3, 2] = float("nan") if which % 2 else float("inf")
        with pytest.raises(AlqError, match="1 logits, embedding, anchor or weight entries are not finite"):
            eng.alfamix_rho(*args)
    with pytest.raises(AlqError, match="C=1"):
        eng.alfamix_rho(logits[:, :1], emb, anc[:1], w[:1])
    with pytest.raises(AlqError, match="alfamix_rho: need"):
        eng.alfamix_rho(logits, emb, anc, w[:, :8].repeat(1, 3))
    with pytest.raises(AlqError, match="alfamix_rho: need"):
        eng.alfamix_rho(logits[:100], emb, anc, w)
    with pytest.raises(AlqError, match="d % 4 == 0"):
        eng.kmeans_nearest(torch.zeros(10, 6, device="cuda"), torch.zeros(10, dtype=torch.int32, device="cuda"),
                           torch.zeros(2, 6, device="cuda"))
    s, *_ = _e2e(eng, 500, 16, 4, 10, 1)
    s.idxs_lb[:] = False
    with pytest.raises(ValueError, match="ALFAMixSampler needs labeled rows"):
        s.query(10)
    lg, em, an, wn = (rng.normal(size=sh).astype(np.float32) for sh in ((300, 10), (300, 16), (10, 16), (10, 16)))
    _check_rho(eng, lg, em, an, wn)
