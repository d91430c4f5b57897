"""ProbCoverSampler on the H100 (K13, K14) against the NumPy statement in probcover_oracle.py."""
import numpy as np
import pytest
import torch

import probcover_oracle as P
from helpers import make_strategy

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from active_learning_b200.engine import Engine
    return Engine()


def _rows(n, d, seed):
    """Basis rows scaled by powers of two (their distances are exactly sqrt(2) after normalisation), a zero row, duplicates
    and random rows."""
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(n, d)).astype(np.float32)
    k = min(n, d, 40)
    x[:k] = 0
    x[np.arange(k), np.arange(k)] = np.float32(2.0) ** (np.arange(k) % 7 - 3)
    if n > k + 2:
        x[k] = 0
    if n > 60:
        x[50:60] = x[45]
    return x


def _csr_host(row_ptr, cols):
    return row_ptr.cpu().numpy(), cols.cpu().numpy()


def _assert_graph(eng, x, delta):
    row_ptr, cols, rech = eng.probcover_graph(torch.from_numpy(x).cuda(), delta)
    rp, cl = _csr_host(row_ptr, cols)
    want_rp, want_cl = P.graph(P.normalize(x), delta)
    assert rp.tolist() == want_rp.tolist() and cl.tolist() == want_cl.tolist()
    return rech


@pytest.mark.parametrize("n", [1, 2, 127, 128, 129, 5000])
@pytest.mark.parametrize("d", [4, 64, 2048])
def test_graph_equals_the_oracle(eng, n, d):
    x = _rows(n, d, n + d)
    s2 = float(np.sqrt(2.0))
    rech = 0
    for delta in (s2, np.nextafter(s2, 3.0), np.nextafter(s2, 0.0), 0.9):
        rech += _assert_graph(eng, x, float(delta))
    if n == 5000:
        # a radius at the random rows' typical distance puts pairs inside the screen's band
        xh = P.normalize(x).astype(np.float64)
        med = float(np.median(np.sqrt(np.maximum(2 - 2 * (xh[100:300] @ xh[300:500].T), 0))))
        rech = _assert_graph(eng, x, med)
        assert rech > 0


def _graph_host(eng, x, delta):
    row_ptr, cols, _ = eng.probcover_graph(torch.from_numpy(x).cuda(), delta)
    return row_ptr, cols, *_csr_host(row_ptr, cols)


def _clustered(n, d, per, seed, noise=0.02):
    rng = np.random.default_rng(seed)
    c = rng.normal(size=(-(-n // per), d)).astype(np.float32)
    x = np.repeat(c, per, axis=0)[:n] + (rng.normal(size=(n, d)) * noise).astype(np.float32)
    return x[rng.permutation(n)]


@pytest.mark.parametrize("case", ["random", "duplicates", "cold", "full_cover", "budget_is_available"])
def test_greedy_equals_the_oracle(eng, case):
    n, d = 40000, 64
    x = _clustered(n, d, 7, 1)
    rng = np.random.default_rng(2)
    if case == "duplicates":                       # equal balls far apart: degree ties across CTA segments
        src = rng.choice(n, 300, replace=False)
        for s in src:
            x[rng.choice(n, 5, replace=False)] = x[s]
    delta = 0.5 if case != "full_cover" else 0.7
    row_ptr, cols, rp, cl = _graph_host(eng, x, delta)
    lab = rng.random(n) < (0.0 if case == "cold" else 0.05)
    avail = ~lab
    budget = {"random": 3000, "duplicates": 3000, "cold": 2000, "full_cover": 20000,
              "budget_is_available": int(avail.sum())}[case]
    picks, steps = eng.probcover_select(row_ptr, cols, torch.from_numpy(lab.astype(np.uint8)).cuda(), budget)
    want = P.greedy(rp, cl, lab, budget)
    assert picks.tolist() == want.tolist() and steps == len(want)
    if case in ("full_cover", "budget_is_available"):
        assert steps < budget                      # coverage ends the greedy: the rest is the host's random fill


def _e2e_strategy(eng, n, d, cache, seed=0):
    rng = np.random.default_rng(seed)
    emb = torch.from_numpy(_clustered(n, d, 5, seed, noise=0.05))
    ev = rng.choice(n, 50, replace=False)
    lab = rng.choice(np.setdiff1d(np.arange(n), ev), 40, replace=False)
    s = make_strategy("ProbCoverSampler", torch.zeros(n, 4), emb, ev, lab, 256, engine=eng, delta=0.45,
                      freeze_feature=cache)
    return s, emb


@pytest.mark.parametrize("cache", [True, False])
def test_query_equals_the_oracle_over_two_rounds(eng, cache):
    s, emb = _e2e_strategy(eng, 6000, 36, cache)
    builds = []
    real = eng.probcover_graph
    eng.probcover_graph = lambda *a, **k: builds.append(1) or real(*a, **k)
    try:
        for rnd in range(2):
            np.random.seed(100 + rnd)
            state = np.random.get_state()
            got, k = s.query(400)
            after = np.random.get_state()
            np.random.set_state(state)
            union = np.asarray(s.get_idxs_for_coreset(), dtype=np.int64)
            is_lab = s.already_labeled_idxs(boolean=True)[union]
            avail = s.available_query_idxs(boolean=True)[union]
            want = union[P.query_positions(emb.numpy()[union], is_lab, avail, 400, 0.45)].tolist()
            assert got == want and k == 400
            assert (np.random.get_state()[1] == after[1]).all() and np.random.get_state()[2] == after[2]
            s.update(got, k)
            s.round += 1
    finally:
        del eng.probcover_graph
    assert len(builds) == (1 if cache else 2)                # the cached round runs K14 only


def test_full_coverage_before_the_budget_fills_at_random(eng):
    s, emb = _e2e_strategy(eng, 3000, 36, True, seed=4)
    s.delta = 1.9                                            # a few balls cover everything
    np.random.seed(7)
    got, k = s.query(500)
    state = np.random.get_state()
    np.random.seed(7)
    union = np.asarray(s.get_idxs_for_coreset(), dtype=np.int64)
    is_lab = s.already_labeled_idxs(boolean=True)[union]
    avail = s.available_query_idxs(boolean=True)[union]
    want = union[P.query_positions(emb.numpy()[union], is_lab, avail, 500, 1.9)].tolist()
    assert got == want and k == 500 and len(set(got)) == 500
    assert (np.random.get_state()[1] == state[1]).all() and np.random.get_state()[2] == state[2]


def test_imagenet_scale_rows_and_picks(eng):
    n, d = 130000, 2048
    x = _clustered(n, d, 10, 9, noise=0.012)
    row_ptr, cols, rp, cl = _graph_host(eng, x, 0.8)
    rng = np.random.default_rng(3)
    rows = rng.choice(n, 64, replace=False)
    want = P.ball_rows(P.normalize(x), 0.8, rows)
    for r, w in zip(rows, want):
        assert cl[rp[r]:rp[r + 1]].tolist() == w.tolist()
    lab = rng.random(n) < 0.01
    picks, steps = eng.probcover_select(row_ptr, cols, torch.from_numpy(lab.astype(np.uint8)).cuda(), 5000)
    assert picks.tolist() == P.greedy(rp, cl, lab, 5000).tolist()


def test_errors_are_clean_and_leave_the_context_usable(eng):
    from active_learning_b200._lib import AlqError
    x = torch.randn(300, 16, device="cuda")
    for bad in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            eng.probcover_graph(x, bad)
    y = x.clone()
    y[7, 3] = float("nan")
    with pytest.raises(ValueError):
        eng.probcover_graph(y, 0.5)
    with pytest.raises(ValueError):
        eng.probcover_graph(torch.empty(0, 16, device="cuda"), 0.5)
    eng._ward_free_bytes = lambda: 1 << 20
    try:
        with pytest.raises(AlqError, match=r"n=300 .* nnz=\d+"):
            eng.probcover_graph(x, 0.5)
    finally:
        del eng._ward_free_bytes
    xn = x.cpu().numpy()
    _assert_graph(eng, xn, 1.0)
