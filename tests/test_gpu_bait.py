"""BAITSampler on the H100 (K24, K25, K26) against the NumPy statement in bait_oracle.py."""
import numpy as np
import pytest
import torch

import bait_oracle as O
from helpers import make_strategy

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from active_learning_b200.engine import Engine
    return Engine()


def _pool(n, d, c, seed, scale=1.0):
    """Embeddings and the logits of a random linear head on them (a spread of confident and unsure rows)."""
    rng = np.random.default_rng(seed)
    h = rng.normal(size=(n, d)).astype(np.float32)
    w = rng.normal(size=(d, c)) * (scale / np.sqrt(d))
    z = (h.astype(np.float64) @ w + rng.normal(size=(n, c)) * 0.5).astype(np.float32)
    return z, h


def _cuda(*a):
    return [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in a]


def test_fisher_equals_the_oracle_within_the_reordered_sum_bound(eng):
    n, d, c = 3000, 64, 10
    z, h = _pool(n, d, c, 1)
    p, F = eng.bait_fisher(*_cuda(z, h))
    Fh = F.cpu().numpy()
    assert (Fh == Fh.T).all()
    want = O.fisher(z, h)
    assert np.abs(p.cpu().numpy() - O.probs(z)).max() <= 1e-15
    # both sides sum the same n products in different orders: each is within (n + 2) u sum |w h h| of the exact value
    pr = O.probs(z)
    ha = np.abs(h.astype(np.float64))
    bound = np.zeros_like(want)
    for a in range(c):
        for b in range(c):
            wab = np.abs((pr[:, a] if a == b else 0.0) - pr[:, a] * pr[:, b]) / n
            bound[a * d:(a + 1) * d, b * d:(b + 1) * d] = ha.T @ (wab[:, None] * ha)
    bound *= 2 * (n + 4) * 2.0 ** -53
    assert (np.abs(Fh - want) <= bound).all()


def _select(eng, z, h, is_lab, avail, budget, lamb=1.0):
    zt, ht = _cuda(z, h)
    p, F = eng.bait_fisher(zt, ht)
    state = eng.bait_init(ht, F, lamb)
    return eng.bait_select(ht, p, F, state, np.flatnonzero(is_lab), np.flatnonzero(avail), budget)


@pytest.mark.parametrize("n,d,n_lab,budget,seed", [(3000, 64, 0, 20, 2), (3000, 64, 300, 20, 3), (8000, 128, 0, 12, 4),
                                                   (8000, 128, 60, 12, 5)])
def test_select_equals_the_oracle(eng, n, d, n_lab, budget, seed):
    c = 10
    z, h = _pool(n, d, c, seed)
    rng = np.random.default_rng(seed)
    is_lab = np.zeros(n, dtype=bool)
    is_lab[rng.choice(n, n_lab, replace=False)] = True
    avail = ~is_lab
    picks, _, fwd, bwd = _select(eng, z, h, is_lab, avail, budget)
    want, wf, wb = O.select(z, h, is_lab, avail, budget)
    assert all(O.separated(s) for s in wf + wb)
    assert picks.tolist() == want.tolist()
    assert len(fwd) == 2 * budget and len(bwd) == budget
    for got, steps in ((fwd, wf), (bwd, wb)):
        best = np.array([max(s.values()) for s in steps])
        assert np.all(np.abs(got - best) <= 1e-9 * np.abs(best))


def _kron_block(rows_p, rows_h, scale2, c, d):
    """sum over the rows of scale2 (diag p - p p^T) (x) h h^T, [C D, C D] (torch fp64)."""
    out = torch.zeros((c * d, c * d), dtype=torch.float64, device="cuda")
    for a in range(c):
        for b in range(a, c):
            w = ((rows_p[:, a] if a == b else 0.0) - rows_p[:, a] * rows_p[:, b]) * scale2
            blk = rows_h.T @ (w[:, None] * rows_h)
            out[a * d:(a + 1) * d, b * d:(b + 1) * d] = blk
            out[b * d:(b + 1) * d, a * d:(a + 1) * d] = blk.T
    return out


def _literal_score(A, F, p, h, s, x):
    """tr((Vt A F A Vt^T)(I + Vt A Vt^T)^-1) of row x with V materialised (torch fp64)."""
    px = p[x]
    R = torch.sqrt(px)[:, None] * (torch.eye(len(px), dtype=torch.float64, device="cuda") - px[None, :])
    V = s * torch.kron(R, h[x][None, :])
    VA = V @ A
    inner = torch.linalg.inv(torch.eye(len(px), dtype=torch.float64, device="cuda") + VA @ V.T)
    return float(torch.trace(VA @ F @ VA.T @ inner))


def test_cifar10_shape_picks_the_budget_and_its_scores_match_a_dense_inverse(eng):
    n, d, c, n_lab, budget = 50000, 512, 10, 5000, 1000
    eng.bait_guard(n, c, d)
    z, h = _pool(n, d, c, 6, scale=3.0)
    rng = np.random.default_rng(6)
    is_lab = np.zeros(n, dtype=bool)
    is_lab[rng.choice(n, n_lab, replace=False)] = True
    avail = ~is_lab
    zt, ht = _cuda(z, h)
    p, F = eng.bait_fisher(zt, ht)
    state = eng.bait_init(ht, F, 1.0)
    picks, order, fwd, bwd = eng.bait_select(ht, p, F, state, np.flatnonzero(is_lab), np.flatnonzero(avail), budget)
    del state
    assert len(picks) == budget and len(set(picks.tolist())) == budget and avail[picks].all()
    assert len(order) == 2 * budget and len(set(order.tolist())) == 2 * budget and np.isin(picks, order).all()
    assert picks.tolist() == [x for x in order.tolist() if x in set(picks.tolist())]
    assert np.isfinite(fwd).all() and len(bwd) == budget and np.isfinite(bwd).all()
    # the scores of forward steps 0, 1, 2 and the last, from M = M0 + the earlier picks' Fisher inverted densely
    s_lab, s = O.scales(n_lab, budget)
    hd = ht.double()
    lab = torch.from_numpy(np.flatnonzero(is_lab)).cuda()
    M0 = _kron_block(p[lab], hd[lab], s_lab ** 2, c, d) + torch.eye(c * d, dtype=torch.float64, device="cuda")
    cand = torch.from_numpy(np.flatnonzero(avail)).cuda()
    A = torch.linalg.inv(M0)
    others = cand[torch.randperm(len(cand), generator=torch.Generator().manual_seed(0))[:64].cuda()]
    lit0 = _literal_score(A, F, p, hd, s, int(order[0]))
    assert abs(lit0 - fwd[0]) <= 1e-9 * abs(lit0)
    assert all(_literal_score(A, F, p, hd, s, int(x)) <= lit0 * (1 + 1e-9) for x in others.tolist())
    for t in (1, 2, 2 * budget - 1):
        prev = torch.from_numpy(order[:t]).cuda()
        M = M0 + _kron_block(p[prev], hd[prev], s ** 2, c, d)
        lit = _literal_score(torch.linalg.inv(M), F, p, hd, s, int(order[t]))
        assert abs(lit - fwd[t]) <= 1e-9 * abs(lit), (t, lit, fwd[t])
    del M, A, M0, F, p
    torch.cuda.empty_cache()


def test_sampler_equals_the_oracle_over_two_rounds(eng):
    n, d, c, budget = 1500, 32, 10, 15
    z, h = _pool(n, d, c, 7)
    rng = np.random.default_rng(7)
    ev = rng.choice(n, 50, replace=False)
    lab = rng.choice(np.setdiff1d(np.arange(n), ev), 40, replace=False)
    s = make_strategy("BAITSampler", torch.from_numpy(z), torch.from_numpy(h), ev, lab, 256, lamb=0.5)
    s.set_engine(eng)
    for rnd in range(2):
        np.random.seed(300 + rnd)
        state = np.random.get_state()
        got, k = s.query(budget)
        after = np.random.get_state()
        np.random.set_state(state)
        union = np.asarray(s.get_idxs_for_coreset(), dtype=np.int64)
        is_lab = s.already_labeled_idxs(boolean=True)[union]
        avail = s.available_query_idxs(boolean=True)[union]
        want = union[O.query_positions(z[union], h[union], is_lab, avail, budget, 0.5)].tolist()
        assert got == want and k == budget
        assert (np.random.get_state()[1] == after[1]).all() and np.random.get_state()[2] == after[2]
        s.update(got, k)
        s.round += 1


def test_errors_are_clean_and_leave_the_context_usable(eng):
    from active_learning_b200._lib import AlqError
    before = torch.cuda.memory_allocated()
    with pytest.raises(AlqError, match=r"bait: n=100 .*need \d+ bytes.*C=1000 classes x D=2048.*\d+ are free"):
        eng.bait_guard(100, 1000, 2048)
    zb, hb = torch.zeros(100, 1000, device="cuda"), torch.zeros(100, 2048, device="cuda")
    mid = torch.cuda.memory_allocated()
    with pytest.raises(AlqError, match=r"C=1000 classes x D=2048"):
        eng.bait_fisher(zb, hb)
    assert torch.cuda.memory_allocated() == mid
    del zb, hb
    assert torch.cuda.memory_allocated() == before
    with pytest.raises(AlqError, match=r"C=17 classes outside"):
        eng.bait_guard(100, 17, 8)
    z, h = _pool(300, 16, 4, 8)
    for bad_z, bad_h in ((True, False), (False, True)):
        zz, hh = z.copy(), h.copy()
        if bad_z:
            zz[7, 1] = np.nan
            zz[90, 0] = np.inf
        else:
            hh[7, 3] = np.nan
            hh[90, 0] = -np.inf
        with pytest.raises(AlqError, match=r"ALQ_ERR_NUMERIC.*2 rows"):
            eng.bait_fisher(*_cuda(zz, hh))
    zt, ht = _cuda(z, h)
    p, F = eng.bait_fisher(zt, ht)
    for bad in (0.0, -1.0, float("nan"), float("inf"), "x"):
        with pytest.raises(ValueError):
            eng.bait_init(ht, F, bad)
        with pytest.raises(ValueError):
            make_strategy("BAITSampler", torch.from_numpy(z), torch.from_numpy(h), [], [], 32, engine=eng, lamb=bad)
    is_lab = np.zeros(300, dtype=bool)
    is_lab[:5] = True
    picks = _select(eng, z, h, is_lab, ~is_lab, 8)[0]
    assert picks.tolist() == O.select(z, h, is_lab, ~is_lab, 8)[0].tolist()
