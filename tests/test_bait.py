"""BAITSampler without a GPU: the oracle's factored, incremental selection against its literal transcription, the
Kronecker identity, the labeled absorption against a dense inverse, the lamb validation, the memory rule, and the
sampler's host logic (pool, RNG draws, budget clamp) through a fake engine built on the oracle."""
import numpy as np
import pytest
import torch

import bait_oracle as O
from helpers import OracleEngine, make_strategy


def _fixture(seed, n, c, d, frac_lab, dup=False):
    """(logits, emb, is_lab, avail): a random linear head on random rows; with dup, groups of exactly equal rows."""
    rng = np.random.default_rng(seed)
    h = rng.normal(size=(n, d)).astype(np.float32)
    z = (h.astype(np.float64) @ rng.normal(size=(d, c)) + rng.normal(size=(n, c))).astype(np.float32)
    is_lab = rng.random(n) < frac_lab
    if dup:                                   # copies of the first forward pick, below and above it: an exact tie
        f0 = O.select(z, h, is_lab, ~is_lab, 1)[1][0]
        src = max(f0, key=f0.get)
        dst = rng.choice(np.flatnonzero(~is_lab & (np.arange(n) != src)), 3, replace=False)
        h[dst], z[dst] = h[src], z[src]
    return z, h, is_lab, ~is_lab


def _separated_run(z, h, is_lab, avail, budget, lamb=1.0):
    """The literal run of a fixture; refuses (fails) a fixture whose top two scores of some step are closer than 1e-8
    relative without being equal."""
    got = O.literal_select(z, h, is_lab, avail, budget, lamb)
    assert all(O.separated(s) for s in got[1] + got[2]), "fixture not separated: choose another seed"
    return got


def _close(a, b, rel=1e-9):
    return all(abs(a[k] - b[k]) <= rel * abs(a[k]) for k in a)


CASES = [  # seed, n, C, D, labeled share, budget, duplicates
    (0, 60, 3, 4, 0.0, 6, False),
    (1, 60, 3, 4, 0.2, 6, False),
    (2, 50, 4, 5, 0.3, 30, False),       # 2B > #candidates
    (3, 40, 3, 3, 0.25, 10 ** 6, False),  # B = #candidates: no backward pass
    (4, 70, 3, 4, 0.1, 8, True),          # exact ties
    (5, 45, 5, 3, 0.0, 12, True),
]


@pytest.mark.parametrize("seed,n,c,d,frac,budget,dup", CASES)
def test_factored_form_equals_the_literal_transcription(seed, n, c, d, frac, budget, dup):
    z, h, is_lab, avail = _fixture(seed, n, c, d, frac, dup)
    budget = min(budget, int(avail.sum()))
    lit, lf, lb = _separated_run(z, h, is_lab, avail, budget)
    inc, f, b = O.select(z, h, is_lab, avail, budget)
    assert inc.tolist() == lit.tolist() and len(inc) == budget and avail[inc].all()
    assert len(f) == O.steps(avail.sum(), budget) and len(b) == len(f) - budget
    assert all(set(x) == set(y) and _close(x, y) for x, y in zip(lf + lb, f + b))
    if dup:                                   # the fixture ties exactly, and a tie goes to the lowest position
        ties = [s for s in f if sum(v == max(s.values()) for v in s.values()) > 1]
        assert ties
        for s, x in zip(f, _forward_order(z, h, is_lab, avail, budget)):
            top = max(s.values())
            assert x == min(k for k, v in s.items() if v == top)


def _forward_order(z, h, is_lab, avail, budget):
    """The forward picks of the incremental form in order (the argmax of each step's scores)."""
    return [max(s, key=lambda k: (s[k], -k)) for s in O.select(z, h, is_lab, avail, budget)[1]]


def test_kronecker_identity():
    z, h, _, _ = _fixture(7, 5, 4, 6, 0.0)
    p = O.probs(z)
    for x in range(5):
        V = O.v_matrix(p[x], h[x])
        hx = h[x].astype(np.float64)
        want = np.kron(np.diag(p[x]) - np.outer(p[x], p[x]), np.outer(hx, hx))
        assert np.allclose(V.T @ V, want, rtol=1e-13, atol=1e-15)
        # row k is sqrt(p_k) (e_k - p) (x) h
        k = 2
        assert np.allclose(V[k], np.kron(np.sqrt(p[x][k]) * (np.eye(4)[k] - p[x]), hx), rtol=1e-14, atol=0)
    F = O.fisher(z, h)
    want = sum(O.v_matrix(p[x], h[x]).T @ O.v_matrix(p[x], h[x]) for x in range(5)) / 5
    assert np.allclose(F, want, rtol=1e-12, atol=1e-15) and (F == F.T).all()


@pytest.mark.parametrize("lamb", [1.0, 0.3, 4.0])
def test_labeled_absorption_equals_the_dense_inverse(lamb):
    z, h, is_lab, _ = _fixture(8, 40, 3, 4, 0.4)
    budget = 7
    p = O.probs(z)
    hh = h.astype(np.float64)
    F = O.fisher(z, h)
    A, At, Gt = O.initial_forms(h, F, lamb)
    st = {"A": A, "At": At, "Gt": Gt, "F": F, "p": p, "h": hh}
    lab = np.flatnonzero(is_lab)
    s_lab, _ = O.scales(len(lab), budget)
    for l in lab:
        O.absorb(st, l, s_lab, 1.0)
    M0 = lamb * np.eye(F.shape[0]) + sum(O.v_matrix(p[l], h[l]).T @ O.v_matrix(p[l], h[l]) for l in lab) / (len(lab) + budget)
    Ainv = np.linalg.inv(M0)
    assert np.allclose(st["A"], Ainv, rtol=1e-10, atol=1e-13)
    # the forms equal h^T A_ab h and h^T (A F A)_ab h of the dense inverse
    d = h.shape[1]
    AFA = Ainv @ F @ Ainv
    wa = np.einsum("xd,adbe,xe->xab", hh, Ainv.reshape(3, d, 3, d), hh)
    wg = np.einsum("xd,adbe,xe->xab", hh, AFA.reshape(3, d, 3, d), hh)
    assert np.allclose(st["At"], wa, rtol=1e-10, atol=1e-13) and np.allclose(st["Gt"], wg, rtol=1e-10, atol=1e-15)


@pytest.mark.parametrize("lamb", [0.0, -1.0, float("nan"), float("inf"), "x", None])
def test_lamb_must_be_finite_and_positive(lamb):
    z, h, ev, lab = _pool()
    with pytest.raises(ValueError):
        make_strategy("BAITSampler", torch.from_numpy(z), torch.from_numpy(h), ev, lab, 32, engine=BaitEngine(),
                      lamb=lamb)
    with pytest.raises(ValueError):
        O.bait_lamb(lamb)


def test_lamb_defaults_to_one():
    from active_learning_b200.query_strategies.bait import bait_lamb
    z, h, ev, lab = _pool()
    s = make_strategy("BAITSampler", torch.from_numpy(z), torch.from_numpy(h), ev, lab, 32, engine=BaitEngine())
    assert s.lamb == 1.0 and bait_lamb(0.25) == O.bait_lamb(0.25) == 0.25


def test_memory_rule_fits_cifar10_and_refuses_imagenet_before_allocating():
    from active_learning_b200._lib import AlqError
    from active_learning_b200.engine import Engine
    for n, c, d in ((50000, 10, 512), (50000, 10, 2048), (1000, 1000, 2048)):
        assert Engine.bait_bytes(n, c, d) == O.bait_bytes(n, c, d) == 24 * (c * d) ** 2 + 16 * n * c * c
    card = 81559 * 2 ** 20                                             # an H100 80GB's whole memory
    eng = Engine.__new__(Engine)
    eng._ward_free_bytes = lambda: card - (1 << 30)
    eng.bait_guard(50000, 10, 512)
    eng.bait_guard(50000, 10, 2048)
    with pytest.raises(AlqError, match=r"bait: n=1281167 rows need \d+ bytes .*C=1000 classes x D=2048.*\d+ are free"):
        eng.bait_guard(1281167, 1000, 2048)
    with pytest.raises(AlqError, match=r"C=17 classes outside \[2, 16\]"):
        eng.bait_guard(1000, 17, 64)


# ---- the sampler's host logic ------------------------------------------------------------------------------------------
class BaitEngine(OracleEngine):
    """The oracle engine plus K24 / K25 / K26 by the NumPy statement; records the calls."""

    def __init__(self, free=None):
        self.calls = []
        self.free = free

    def bait_guard(self, n, c, d):
        self.calls.append(("guard", n, c, d))
        if self.free is not None and O.bait_bytes(n, c, d) > self.free:
            from active_learning_b200._lib import AlqError
            raise AlqError(f"bait: n={n}")

    def bait_fisher(self, logits, emb):
        self.calls.append("fisher")
        self._z = logits.numpy()
        return torch.from_numpy(O.probs(self._z)), torch.from_numpy(O.fisher(self._z, emb.numpy()))

    def bait_init(self, emb, F, lamb):
        self.calls.append("init")
        return O.initial_forms(emb.numpy(), F.numpy(), lamb), lamb

    def bait_select(self, emb, p, F, state, lab_pos, cand_pos, budget):
        self.calls.append("select")
        n = emb.shape[0]
        is_lab, avail = np.zeros(n, dtype=bool), np.zeros(n, dtype=bool)
        is_lab[lab_pos] = True
        avail[cand_pos] = True
        picks, f, b = O.select(self._z, emb.numpy(), is_lab, avail, budget, state[1], F=F.numpy())
        return picks, picks, np.array([max(s.values()) for s in f]), np.array([max(s.values()) for s in b])


def _pool(n=90, d=4, c=3, seed=3, n_lab=9):
    rng = np.random.default_rng(seed)
    h = rng.normal(size=(n, d)).astype(np.float32)
    z = (h.astype(np.float64) @ rng.normal(size=(d, c))).astype(np.float32)
    eval_idxs = rng.choice(n, 8, replace=False)
    labeled = rng.choice(np.setdiff1d(np.arange(n), eval_idxs), n_lab, replace=False)
    return z, h, eval_idxs, labeled


@pytest.mark.parametrize("budget,n_lab,lamb,kw", [(5, 9, 1.0, {}), (9, 9, 0.5, {}), (10 ** 6, 9, 1.0, {}),
                                                  (6, 0, 2.0, {}), (5, 9, 1.0, {"subset_unlabeled": 30}),
                                                  (5, 9, 1.0, {"subset_labeled": 4})])
def test_query_equals_the_oracle_and_draws_only_the_pool(budget, n_lab, lamb, kw):
    z, h, ev, lab = _pool(n_lab=n_lab)
    eng = BaitEngine()
    s = make_strategy("BAITSampler", torch.from_numpy(z), torch.from_numpy(h), ev, lab, 32, engine=eng, lamb=lamb, **kw)
    for rnd in range(2):
        np.random.seed(21 + rnd)
        got, k = s.query(budget)
        state = np.random.get_state()
        np.random.seed(21 + rnd)
        union = np.asarray(s.get_idxs_for_coreset(), dtype=np.int64)
        is_lab = s.already_labeled_idxs(boolean=True)[union]
        avail = s.available_query_idxs(boolean=True)[union]
        want = union[O.query_positions(z[union], h[union], is_lab, avail, budget, lamb)].tolist()
        assert got == want and k == len(want) == min(budget, int(avail.sum()))
        assert len(set(got)) == k and not s.idxs_lb[got].any() and not np.isin(got, ev).any()
        after = np.random.get_state()                                  # the two shuffles are the only draws
        assert state[2] == after[2] and (state[1] == after[1]).all()
        assert eng.calls[-4][0] == "guard" and eng.calls[-3:] == ["fisher", "init", "select"]
        s.update(got, k)
        s.round += 1


def test_zero_budget_returns_nothing_and_builds_nothing():
    z, h, ev, lab = _pool()
    eng = BaitEngine()
    s = make_strategy("BAITSampler", torch.from_numpy(z), torch.from_numpy(h), ev, lab, 32, engine=eng)
    np.random.seed(5)
    assert s.query(0) == ([], 0)
    state = np.random.get_state()
    np.random.seed(5)
    s.get_idxs_for_coreset()
    assert (np.random.get_state()[1] == state[1]).all() and eng.calls == []


def test_a_pool_beyond_memory_is_refused_before_anything_is_built():
    from active_learning_b200._lib import AlqError
    z, h, ev, lab = _pool()
    eng = BaitEngine(free=1000)
    s = make_strategy("BAITSampler", torch.from_numpy(z), torch.from_numpy(h), ev, lab, 32, engine=eng)
    with pytest.raises(AlqError, match=r"bait: n=82"):
        s.query(5)
    assert [c for c in eng.calls if not isinstance(c, tuple)] == []


def test_registered_for_dispatch_and_drop_in():
    from active_learning_b200.integration import make_drop_in
    from active_learning_b200.query_strategies.bait import BAITQuery
    from active_learning_b200.query_strategies.get_strategy import ACCELERATED, get_strategy
    assert "BAITSampler" in ACCELERATED and get_strategy("BAITSampler").__name__ == "BAITSampler"

    class Base:
        pass

    cls = make_drop_in(Base)["BAITSampler"]
    assert issubclass(cls, BAITQuery) and issubclass(cls, Base)
