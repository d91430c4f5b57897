"""MaxHerdingSampler on the H100 (K22, K23) against the NumPy statement in maxherding_oracle.py."""
import numpy as np
import pytest
import torch

import maxherding_oracle as H
from helpers import make_strategy

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from active_learning_b200.engine import Engine
    return Engine()


def _clustered(n, d, per, seed, noise=0.05, dups=0):
    """Rows around n / per random centres, a zero row and `dups` groups of 5 exact duplicates."""
    rng = np.random.default_rng(seed)
    c = rng.normal(size=(-(-n // per), d)).astype(np.float32)
    x = np.repeat(c, per, axis=0)[:n] + (rng.normal(size=(n, d)) * noise).astype(np.float32)
    x = x[rng.permutation(n)]
    if n > 10:
        x[n // 3] = 0
    for s in rng.choice(n, dups, replace=False):
        x[rng.choice(n, 5, replace=False)] = x[s]
    return x


def _kernel(eng, x, sigma):
    xhat = eng.normalize(torch.from_numpy(x).cuda())
    return xhat, eng.herding_kernel(xhat, sigma)


def _assert_rows_match(K_rows, xhat_host, q, rows):
    """K22's rows against the oracle: equal except where the fp64 value lies within 1 fp64 ulp of an fp32 rounding
    midpoint (CUDA's exp is within 1 ulp), and there within one fp32 ulp."""
    want, e = H.kernel_rows(xhat_host, q, rows)
    diff = K_rows != want
    band = H.f32_midpoint_band(e)
    assert not (diff & ~band).any(), np.argwhere(diff & ~band)[:5]
    assert (np.abs(K_rows[diff].view(np.int32).astype(np.int64) - want[diff].view(np.int32)) <= 1).all()


@pytest.mark.parametrize("n,d,sigma", [(1, 4, 0.5), (65, 36, 0.3), (1000, 128, 0.5), (3000, 128, 0.7), (700, 2048, 1.0),
                                       (3000, 130, 0.05)])
def test_kernel_equals_the_oracle(eng, n, d, sigma):
    x = _clustered(n, d, 6, n + d, dups=n // 200)
    xhat, K = _kernel(eng, x, sigma)
    Kh, xh = K.cpu().numpy(), xhat.cpu().numpy()
    assert (Kh == Kh.T).all() and (np.diag(Kh) == 1.0).all()
    _assert_rows_match(Kh, xh, H.herding_q(sigma), np.arange(n))


def test_kernel_past_2_31_entries(eng):
    n, d = 50000, 512
    x = _clustered(n, d, 10, 1)
    xhat, K = _kernel(eng, x, 0.6)
    assert (torch.diagonal(K) == 1.0).all()
    for lo in range(0, n, 4096):                                       # exact symmetry, a band of rows at a time
        hi = min(n, lo + 4096)
        assert torch.equal(K[lo:hi], K[:, lo:hi].t())
    rows = np.concatenate([np.random.default_rng(2).choice(n, 40, replace=False), [0, n - 1, 46340, 46341]])
    _assert_rows_match(K[torch.from_numpy(rows).cuda()].cpu().numpy(), xhat.cpu().numpy(), H.herding_q(0.6), rows)


@pytest.mark.parametrize("case", ["cold", "labeled", "ties", "underflow", "budget_is_available"])
def test_greedy_equals_the_oracle_bit_for_bit(eng, case):
    n, d = (3000, 32) if case == "budget_is_available" else (8000, 64)
    if case == "underflow":                        # unit rows about sqrt(2) apart: every off-diagonal entry is 0
        x = np.random.default_rng(5).normal(size=(n, d)).astype(np.float32)
    else:
        x = _clustered(n, d, 8, 5, dups=300 if case == "ties" else 0)
    sigma = {"underflow": 0.01}.get(case, 0.4)
    _, K = _kernel(eng, x, sigma)
    if case == "underflow":
        assert torch.equal(K, torch.eye(n, device="cuda"))
    rng = np.random.default_rng(6)
    lab = rng.random(n) < (0.0 if case == "cold" else 0.1)
    avail = ~lab & (rng.random(n) < 0.95)
    budget = int(avail.sum()) if case == "budget_is_available" else 600
    picks, m, sum_s = eng.herding_select(K, torch.from_numpy(lab).cuda(), torch.from_numpy(avail).cuda(), budget)
    Kh = K.cpu().numpy()
    want, want_m = H.greedy(Kh, lab, avail, budget)
    assert picks.tolist() == want.tolist()
    assert torch.equal(m.cpu(), torch.from_numpy(want_m))
    assert sum_s > 0
    if case == "underflow":
        assert picks.tolist() == np.flatnonzero(avail)[:budget].tolist()


def _strategy(n, d, seed, sigma, n_lab):
    rng = np.random.default_rng(seed)
    emb = torch.from_numpy(_clustered(n, d, 6, seed, dups=20))
    ev = rng.choice(n, 50, replace=False)
    lab = rng.choice(np.setdiff1d(np.arange(n), ev), n_lab, replace=False)
    return make_strategy("MaxHerdingSampler", torch.zeros(n, 4), emb, ev, lab, 256, sigma=sigma), emb


def _pool_state(s):
    union = np.asarray(s.get_idxs_for_coreset(), dtype=np.int64)
    return union, s.already_labeled_idxs(boolean=True)[union], s.available_query_idxs(boolean=True)[union]


def test_query_equals_the_oracle_end_to_end_over_two_rounds(eng):
    s, emb = _strategy(3000, 128, 0, 0.5, 30)
    s.set_engine(eng)
    for rnd in range(2):
        np.random.seed(100 + rnd)
        state = np.random.get_state()
        got, k = s.query(200)
        after = np.random.get_state()
        np.random.set_state(state)
        union, is_lab, avail = _pool_state(s)
        want = union[H.query_positions(emb.numpy()[union], is_lab, avail, 200, 0.5)].tolist()
        assert got == want and k == 200
        assert (np.random.get_state()[1] == after[1]).all() and np.random.get_state()[2] == after[2]
        s.update(got, k)
        s.round += 1


def test_query_equals_the_oracles_greedy_on_the_devices_matrix(eng):
    s, emb = _strategy(20000, 512, 1, 0.6, 200)
    s.set_engine(eng)
    seen = []
    real = eng.herding_kernel
    eng.herding_kernel = lambda *a, **k: seen.append(real(*a, **k).cpu().numpy()) or torch.from_numpy(seen[-1]).cuda()
    try:
        for rnd in range(2):
            np.random.seed(200 + rnd)
            state = np.random.get_state()
            got, k = s.query(300)
            after = np.random.get_state()
            np.random.set_state(state)
            union, is_lab, avail = _pool_state(s)
            want = union[H.greedy(seen[-1], is_lab, avail, 300)[0]].tolist()
            assert got == want and k == 300
            assert (np.random.get_state()[1] == after[1]).all()
            s.update(got, k)
            s.round += 1
    finally:
        del eng.herding_kernel


def test_imagenet_lt_shape_fits_and_its_first_picks_maximise_the_literal_gain(eng):
    n, d, budget = 115846, 2048, 10000
    eng.herding_guard(n, d)
    g = torch.Generator(device="cuda").manual_seed(3)
    centres = torch.randn(n // 20 + 1, d, device="cuda", generator=g)
    x = centres[torch.randint(0, centres.shape[0], (n,), device="cuda", generator=g)]
    x += 0.3 * torch.randn(n, d, device="cuda", generator=g)
    xhat = eng.normalize(x)
    del x, centres
    K = eng.herding_kernel(xhat, 0.5)
    del xhat
    rng = np.random.default_rng(4)
    lab = rng.random(n) < 0.1
    avail = ~lab
    picks, m, sum_s = eng.herding_select(K, torch.from_numpy(lab).cuda(), torch.from_numpy(avail).cuda(), budget)
    assert len(picks) == budget and len(set(picks.tolist())) == budget and avail[picks].all()
    lab_rows = torch.from_numpy(np.flatnonzero(lab)).cuda()
    mm = torch.zeros(n, dtype=torch.float32, device="cuda")
    for lo in range(0, len(lab_rows), 2048):
        mm = torch.maximum(mm, K[lab_rows[lo:lo + 2048]].max(dim=0).values)
    cand = torch.from_numpy(avail).cuda()
    for t in range(20):
        lit = torch.zeros(n, dtype=torch.float64, device="cuda")
        for lo in range(0, n, 2048):
            lit += (K[lo:lo + 2048].double() - mm[lo:lo + 2048, None].double()).clamp_min_(0).sum(dim=0)
        best = lit[cand].max().item()
        c = int(picks[t])
        assert lit[c].item() >= best * (1 - 1e-9), (t, lit[c].item(), best)
        mm = torch.maximum(mm, K[c])
        cand[c] = False
    del K
    torch.cuda.empty_cache()


def test_errors_are_clean_and_leave_the_context_usable(eng):
    from active_learning_b200._lib import AlqError
    x = torch.randn(300, 16, device="cuda")
    for bad in (None, 0.0, -1.0, float("nan"), float("inf"), 1e-200, 1e155):
        with pytest.raises(ValueError):
            eng.herding_kernel(x, bad)
    y = x.clone()
    y[7, 3] = float("nan")
    y[90, 0] = float("inf")
    with pytest.raises(AlqError, match=r"ALQ_ERR_NUMERIC.*2 rows"):
        eng.herding_kernel(y, 0.5)
    with pytest.raises(AlqError):
        eng.herding_kernel(torch.empty(0, 16, device="cuda"), 0.5)
    before = torch.cuda.memory_allocated()
    eng._ward_free_bytes = lambda: 1 << 20
    try:
        with pytest.raises(AlqError, match=r"n=300 .*subset_unlabeled"):
            eng.herding_kernel(x, 0.5)
        assert torch.cuda.memory_allocated() == before
    finally:
        del eng._ward_free_bytes
    K = eng.herding_kernel(x, 0.5)
    lab = torch.zeros(300, dtype=torch.uint8, device="cuda")
    with pytest.raises(AlqError):
        eng.herding_select(K[:, :299], lab, lab, 5)
    with pytest.raises(AlqError):
        eng.herding_select(K, lab[:299], lab, 5)
    with pytest.raises(AlqError):
        eng.herding_select(K.double(), lab, lab, 5)
    avail = torch.ones(300, dtype=torch.uint8, device="cuda")
    picks, m, _ = eng.herding_select(K, lab, avail, 10)
    want, want_m = H.greedy(K.cpu().numpy(), np.zeros(300, bool), np.ones(300, bool), 10)
    assert picks.tolist() == want.tolist() and torch.equal(m.cpu(), torch.from_numpy(want_m))
    assert eng.herding_select(K, lab, torch.zeros_like(avail), 10)[0].tolist() == []
