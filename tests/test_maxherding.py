"""MaxHerdingSampler without a GPU: the oracle's incremental greedy against the literal one, its gains against
F(S u {c}) - F(S), the kernel's edge cases, the sigma validation, the memory rule, and the sampler's host logic (pool, RNG
draws, budget clamp) through a fake engine built on the oracle."""
import math

import numpy as np
import pytest
import torch

import maxherding_oracle as H
from helpers import OracleEngine, make_strategy


def _rows(rng, n, d, dup=False, zero=False):
    x = rng.normal(size=(n, d)).astype(np.float32)
    if dup:
        x[rng.integers(0, n, n // 4)] = x[3]                           # duplicated rows: exact ties
        x[rng.integers(0, n, n // 8)] = x[7]
    if zero:
        x[[0, n // 2]] = 0
    return H.normalize(x)


def _gap_ok(gains):
    """The largest gain is either tied exactly or ahead of the next distinct gain by >= 1e-9 relative."""
    g = np.sort(np.array(list(gains.values())))[::-1]
    below = g[g < g[0]]
    return len(below) == 0 or g[0] - below[0] >= 1e-9 * g[0]


CASES = [(0, 0.0, False), (1, 0.1, False), (2, 0.0, True), (3, 0.1, True), (4, 0.3, True), (5, 0.1, False)]


@pytest.mark.parametrize("seed,frac,dup", CASES)
def test_incremental_greedy_equals_the_literal_greedy(seed, frac, dup):
    rng = np.random.default_rng(seed)
    n, d = 120 + 20 * seed, 8
    xh = _rows(rng, n, d, dup=dup, zero=seed == 5)
    K = H.kernel_matrix(xh, H.herding_q(0.6))
    lab = rng.random(n) < frac
    avail = ~lab & (rng.random(n) < 0.9)
    budget = 40
    lit, gains = H.literal_greedy(K, lab, avail, budget)
    assert all(_gap_ok(g) for g in gains)
    inc, m, seen = H.greedy(K, lab, avail, budget, return_gains=True)
    assert inc.tolist() == lit.tolist()
    if dup:
        assert any(sum(v == max(g.values()) for v in g.values()) > 1 for g in gains)   # the fixture does tie
    # the incremental gains against F(S u {c}) - F(S), and m against the literal running max
    mm = H.initial_m(K, lab)
    for t, c in enumerate(inc):
        cols = np.flatnonzero(avail & ~np.isin(np.arange(n), inc[:t]))
        want = H.literal_gains(K, mm, cols)
        got = seen[t][cols]
        assert np.all(np.abs(got - want) <= 1e-12 * np.maximum(np.abs(want), 1.0))
        mm = np.maximum(mm, K[c])
    assert (m == mm).all()


def test_the_kernel_is_symmetric_with_unit_diagonal_and_keeps_zero_rows():
    rng = np.random.default_rng(7)
    xh = _rows(rng, 90, 12, dup=True, zero=True)
    q = H.herding_q(0.8)
    K = H.kernel_matrix(xh, q)
    assert (K == K.T).all() and (np.diag(K) == 1.0).all()
    # a zero row is at squared distance 1 from every unit row (exactly, up to the unit rows' own rounding)
    z = 0
    others = np.flatnonzero(np.abs(xh).sum(axis=1) > 0)
    assert np.allclose(K[z, others], np.float32(math.exp(-1.0 / q)), rtol=1e-6)
    # fp64 values next to an fp32 midpoint are few and the band test finds exact midpoints
    _, e = H.kernel_rows(xh, q, np.arange(10))
    assert H.f32_midpoint_band(e).mean() < 1e-3
    mid = np.float64(np.float32(0.75)) + np.float64(np.spacing(np.float32(0.75))) / 2
    assert H.f32_midpoint_band(np.array([mid, np.nextafter(mid, 1.0), 0.75]))[:2].all()
    assert not H.f32_midpoint_band(np.array([0.75]))[0]


def test_an_underflowed_kernel_picks_by_lowest_position():
    rng = np.random.default_rng(8)
    n = 150
    xh = _rows(rng, n, 16)
    K = H.kernel_matrix(xh, H.herding_q(0.01))
    assert (K == np.eye(n, dtype=np.float32)).all()
    lab = rng.random(n) < 0.1
    avail = ~lab
    picks, m = H.greedy(K, lab, avail, 30)
    assert picks.tolist() == np.flatnonzero(avail)[:30].tolist()
    # every row covered by a duplicate of a labeled row: all gains 0, still the lowest free positions
    x = np.repeat(xh[:1], n, axis=0)
    K1 = H.kernel_matrix(x, H.herding_q(0.5))
    lab1 = np.zeros(n, dtype=bool)
    lab1[5] = True
    picks1, m1 = H.greedy(K1, lab1, ~lab1, 10)
    assert picks1.tolist() == [0, 1, 2, 3, 4, 6, 7, 8, 9, 10] and (m1 == 1.0).all()


def test_a_budget_of_every_candidate_picks_each_once():
    rng = np.random.default_rng(9)
    n = 80
    xh = _rows(rng, n, 6, dup=True)
    K = H.kernel_matrix(xh, H.herding_q(0.5))
    lab = rng.random(n) < 0.2
    avail = ~lab
    picks, m = H.greedy(K, lab, avail, 10 ** 6)
    assert sorted(picks.tolist()) == np.flatnonzero(avail).tolist()
    assert picks.tolist() == H.literal_greedy(K, lab, avail, 10 ** 6)[0].tolist()
    assert (m == 1.0).all()                                            # every row is its own best cover


@pytest.mark.parametrize("sigma", [None, 0.0, -1.0, float("nan"), float("inf"), 1e-200, 1e-155, 1e155])
def test_sigma_is_required_finite_positive_and_gives_a_normal_q(sigma):
    emb, logits, ev, lab = _pool()
    with pytest.raises(ValueError):
        make_strategy("MaxHerdingSampler", logits, emb, ev, lab, 32, engine=HerdingEngine(), sigma=sigma)
    with pytest.raises(ValueError):
        H.herding_q(sigma)


def test_q_is_formed_once_and_alike_in_the_oracle_and_the_sampler():
    from active_learning_b200.query_strategies.maxherding import herding_q
    for s in (1e-150, 0.1, 0.3, 1.0 / 3.0, 1.0, 7.5, 1e150):
        assert herding_q(s) == H.herding_q(s) == 2.0 * s * s


def test_memory_rule_fits_imagenet_lt_on_80_gb_and_refuses_150000_rows():
    from active_learning_b200._lib import AlqError
    from active_learning_b200.engine import Engine
    need = Engine.herding_bytes(115846, 2048)
    assert 4 * 115846 ** 2 < need < 80 * 10 ** 9
    card = 81559 * 2 ** 20                                             # an H100 80GB's whole memory
    assert Engine.herding_bytes(150000, 2048) > card
    eng = Engine.__new__(Engine)
    eng._ward_free_bytes = lambda: card - (1 << 30)
    eng.herding_guard(115846, 2048)
    with pytest.raises(AlqError, match=r"n=150000 .*need \d+ bytes.*\d+ are free.*subset_unlabeled"):
        eng.herding_guard(150000, 2048)


# ---- the sampler's host logic ------------------------------------------------------------------------------------------
class HerdingEngine(OracleEngine):
    """The oracle engine plus K22 / K23 by the NumPy statement; records the calls."""

    def __init__(self, free=None):
        self.calls = []
        self.free = free

    def normalize(self, x):
        self.calls.append("normalize")
        return torch.from_numpy(H.normalize(x.numpy()))

    def herding_guard(self, n, d):
        self.calls.append(("guard", n, d))
        if self.free is not None and 4 * n * n > self.free:
            from active_learning_b200._lib import AlqError
            raise AlqError(f"maxherding: n={n}")

    def herding_kernel(self, xhat, sigma):
        self.calls.append("kernel")
        return torch.from_numpy(H.kernel_matrix(xhat.numpy(), H.herding_q(sigma)))

    def herding_select(self, K, labeled, avail, budget):
        self.calls.append("select")
        picks, m = H.greedy(K.numpy(), labeled.numpy().astype(bool), avail.numpy().astype(bool), budget)
        return picks, torch.from_numpy(m), 0

    def herding_release(self):
        self.calls.append("release")


def _pool(n=160, d=6, seed=3, n_lab=9):
    rng = np.random.default_rng(seed)
    emb = torch.from_numpy(rng.normal(size=(n, d)).astype(np.float32))
    logits = torch.zeros(n, 4)
    eval_idxs = rng.choice(n, 12, replace=False)
    rest = np.setdiff1d(np.arange(n), eval_idxs)
    labeled = rng.choice(rest, n_lab, replace=False)
    return emb, logits, eval_idxs, labeled


def _expected(s, emb, budget, sigma):
    """What the query returns, replayed from the same NumPy state: the two shuffles, then the oracle."""
    union = np.asarray(s.get_idxs_for_coreset(), dtype=np.int64)
    is_lab = s.already_labeled_idxs(boolean=True)[union]
    avail = s.available_query_idxs(boolean=True)[union]
    return union[H.query_positions(emb.numpy()[union], is_lab, avail, budget, sigma)].tolist()


@pytest.mark.parametrize("sigma,budget,n_lab,kw", [(0.5, 7, 9, {}), (1.0, 25, 9, {}), (0.02, 11, 9, {}),
                                                   (0.7, 10 ** 6, 9, {}), (0.7, 20, 0, {}),
                                                   (0.7, 15, 9, {"subset_unlabeled": 60}),
                                                   (0.7, 15, 9, {"subset_labeled": 4})])
def test_query_equals_the_oracle_and_draws_only_the_pool(sigma, budget, n_lab, kw):
    emb, logits, ev, lab = _pool(n_lab=n_lab)
    eng = HerdingEngine()
    s = make_strategy("MaxHerdingSampler", logits, emb, ev, lab, 32, engine=eng, sigma=sigma, **kw)
    for rnd in range(2):
        np.random.seed(11 + rnd)
        got, k = s.query(budget)
        state = np.random.get_state()
        np.random.seed(11 + rnd)
        want = _expected(s, emb, budget, sigma)
        assert got == want and k == len(want)
        avail_total = int(s.available_query_idxs(boolean=True).sum())
        assert k == min(budget, avail_total) or kw
        assert len(set(got)) == k and not s.idxs_lb[got].any() and not np.isin(got, ev).any()
        after = np.random.get_state()                                  # the two shuffles are the only draws
        assert state[2] == after[2] and (state[1] == after[1]).all()
        assert eng.calls[-5][0] == "guard" and eng.calls[-4:] == ["normalize", "kernel", "select", "release"]
        if k:
            s.update(got, k)
            s.round += 1


def test_zero_budget_returns_nothing_and_builds_nothing():
    emb, logits, ev, lab = _pool()
    eng = HerdingEngine()
    s = make_strategy("MaxHerdingSampler", logits, emb, ev, lab, 32, engine=eng, sigma=0.7)
    np.random.seed(5)
    assert s.query(0) == ([], 0)
    state = np.random.get_state()
    np.random.seed(5)
    s.get_idxs_for_coreset()
    assert (np.random.get_state()[1] == state[1]).all() and eng.calls == []


def test_a_pool_beyond_memory_is_refused_before_anything_is_built():
    from active_learning_b200._lib import AlqError
    emb, logits, ev, lab = _pool()
    eng = HerdingEngine(free=1000)
    s = make_strategy("MaxHerdingSampler", logits, emb, ev, lab, 32, engine=eng, sigma=0.7)
    with pytest.raises(AlqError, match=r"maxherding: n=148"):
        s.query(5)
    assert [c for c in eng.calls if not isinstance(c, tuple)] == []


def test_registered_for_dispatch_and_drop_in():
    from active_learning_b200.integration import make_drop_in
    from active_learning_b200.query_strategies.get_strategy import ACCELERATED, get_strategy
    from active_learning_b200.query_strategies.maxherding import MaxHerdingQuery
    assert "MaxHerdingSampler" in ACCELERATED and get_strategy("MaxHerdingSampler").__name__ == "MaxHerdingSampler"

    class Base:
        pass

    cls = make_drop_in(Base)["MaxHerdingSampler"]
    assert issubclass(cls, MaxHerdingQuery) and issubclass(cls, Base)
