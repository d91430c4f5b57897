"""K11, the persistent BalancingSampler loop, on the CPU: its NumPy twin (tests/balancing_loop_oracle.py) against NumPy's
own RNG, torch's imbalance test, the oracle and the picks the reference itself produced, and the sampler's routing
through an engine whose `balancing_select` is the twin."""
import os
import pickle
import re

import numpy as np
import pytest
import torch

from balancing_loop_oracle import MT19937Twin, balancing_loop, needs_balancing
from helpers import OracleEngine
from oracle import al_oracle as O
from test_balancing import balancing_strategy, bgold, masks  # noqa: F401  (fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lgold():
    return dict(np.load(os.path.join(ROOT, "tests", "golden", "reference_golden_balancing_loop.npz")))


def _state_equal(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and a[2] == b[2] and a[3] == b[3] and a[4] == b[4]


RANGES = [1, 2, 3] + [v for k in range(1, 22) for v in (2 ** k, 2 ** k + 1)]


@pytest.mark.parametrize("pos", [0, 300, 620, 623, 624])
def test_twin_draws_equal_numpy_choice(pos):
    np.random.seed(pos + 5)
    np.random.random_sample(700)                   # a twisted state
    name, key, _, g, cg = np.random.get_state()
    np.random.set_state((name, key, pos, g, cg))   # the next draws cross the twist at position 624
    for n in RANGES:
        tw = MT19937Twin(np.random.get_state())
        a = np.arange(n)
        got = [tw.bounded(n - 1) for _ in range(4)]
        want = [int(np.random.choice(a)) for _ in range(4)]
        assert got == want, n
        assert _state_equal(tw.state(), np.random.get_state()), n
        if n == 1:
            assert tw.outputs == 0                 # rng == 0 draws nothing


def _histograms():
    rng = np.random.default_rng(2)
    for _ in range(10000):
        c = int(rng.integers(1, 16))
        kind = rng.integers(6)
        if kind == 0:
            h = np.full(c, int(rng.integers(0, 100)))
        elif kind == 1:
            h = rng.integers(0, 3, size=c) * int(rng.integers(0, 5))
        elif kind == 2:
            h = (2 ** 24 // c - 64) + rng.integers(-64, 64, size=c)
        else:
            h = rng.integers(0, 200, size=c)
        yield h.astype(np.int64), int(rng.integers(1, 400))
    yield np.array([7]), 1                          # a single class
    yield np.zeros(10, dtype=np.int64), 5


def test_fp32_imbalance_test_equals_torch():
    from active_learning_b200.query_strategies.balancing import BalancingQuery
    n = 0
    for h, rem in _histograms():
        want = BalancingQuery._needs_balancing(torch.from_numpy(h), rem)
        got = needs_balancing(h, rem)
        assert (got is None) == (want is None), (h, rem)
        if got is not None:
            assert np.array_equal(got, want.numpy()), (h, rem)
        n += 1
    assert n >= 10000


def _run_twin(g, tag):
    avail, lb = masks(g, tag)
    np.random.seed(int(g.get(f"{tag}_seed", 11)))
    out = balancing_loop(g[f"{tag}_emb"], g[f"{tag}_ys"], avail, lb, int(g[f"{tag}_classes"]), int(g[f"{tag}_budget"]))
    np.random.set_state(out["state"])
    return out, np.random.random_sample()


@pytest.mark.parametrize("tag", ["a", "b"])
def test_twin_matches_oracle_and_reference_on_balancing_goldens(bgold, tag):  # noqa: F811
    g = bgold
    out, after = _run_twin(g, tag)
    assert out["picks"] == g[f"{tag}_picks"].tolist()
    assert out["balancing_steps"] == int(g[f"{tag}_balancing_steps"])
    avail, lb = masks(g, tag)
    np.random.seed(11)
    picks, _ = O.balancing_query(torch.from_numpy(g[f"{tag}_emb"]), torch.from_numpy(g[f"{tag}_ys"]), avail, lb,
                                 float(g[f"{tag}_budget"]), int(g[f"{tag}_classes"]))
    assert picks == out["picks"] and np.random.random_sample() == after


@pytest.mark.parametrize("tag", ["m", "r"])
def test_twin_matches_oracle_and_reference_on_loop_goldens(lgold, tag):
    g = lgold
    out, after = _run_twin(g, tag)
    assert out["picks"] == g[f"{tag}_picks"].tolist() and after == float(g[f"{tag}_after"])
    assert out["balancing_steps"] == int(g[f"{tag}_balancing_steps"])
    switches = int(np.count_nonzero(np.diff(np.array(out["branch"], dtype=int))))
    if tag == "m":
        assert 0 < out["balancing_steps"] < int(g["m_budget"]) and switches >= 4 and out["min_gap"] >= 1e-4
    else:
        assert out["balancing_steps"] == 0 and out["outputs"] > 624
    avail, lb = masks(g, tag)
    np.random.seed(int(g[f"{tag}_seed"]))
    picks, _ = O.balancing_query(torch.from_numpy(g[f"{tag}_emb"]), torch.from_numpy(g[f"{tag}_ys"]), avail, lb,
                                 float(g[f"{tag}_budget"]), int(g[f"{tag}_classes"]))
    assert picks == out["picks"] and np.random.random_sample() == after


def test_twin_rejects_out_of_range_labels(lgold):
    g = lgold
    avail, lb = masks(g, "m")
    ys = g["m_ys"].copy()
    row = int(np.flatnonzero(avail)[7])
    ys[row] = 10
    with pytest.raises(ValueError, match=f"available row {row} has label 10"):
        balancing_loop(g["m_emb"], ys, avail, lb, 10, 5)


class TwinEngine(OracleEngine):
    """OracleEngine plus K11's contract, computed by the twin: declines (None) when C * D floats exceed `centre_floats`,
    the stand-in for the shared-memory limit."""

    def __init__(self, centre_floats=1 << 20):
        self.centre_floats = centre_floats
        self.calls = self.declined = 0

    def balancing_select(self, emb, xn, labels, avail, labeled, num_classes, budget):
        self.calls += 1
        if num_classes * emb.shape[1] > self.centre_floats:
            self.declined += 1
            return None
        out = balancing_loop(emb.numpy(), labels.numpy(), avail.numpy().astype(bool), labeled.numpy().astype(bool),
                             num_classes, budget, np.random.get_state())
        np.random.set_state(out["state"])
        return np.asarray(out["picks"], dtype=np.int64), out["balancing_steps"]


@pytest.mark.parametrize("tag", ["a", "b"])
def test_sampler_routes_through_balancing_select(bgold, tag):  # noqa: F811
    g = bgold
    eng = TwinEngine()
    s = balancing_strategy(g, tag, engine=eng)
    np.random.seed(11)
    idx, cost = s.query(float(g[f"{tag}_budget"]))
    assert eng.calls == 1 and eng.declined == 0
    assert [int(i) for i in idx] == g[f"{tag}_picks"].tolist() and cost == int(g[f"{tag}_budget"])
    assert all(isinstance(i, np.int64) for i in idx)
    after = np.random.random_sample()
    _, want = _run_twin(g, tag)
    assert after == want
    s.update(idx, cost)
    pickle.dumps(s)
    cached = s._bal_cache[0]                       # second round under --freeze_feature: the cached embeddings
    idx2, cost2 = s.query(5.0)
    assert s._bal_cache[0] is cached and cost2 == 5 and eng.calls == 2 and not set(map(int, idx2)) & set(map(int, idx))


def test_sampler_loop_budget_edges(bgold):  # noqa: F811
    g = bgold
    avail, lb = masks(g, "b")
    eng = TwinEngine()
    s = balancing_strategy(g, "b", engine=eng)
    np.random.seed(3)
    idx, cost = s.query(1e9)                       # clamped to the available rows
    assert cost == int(avail.sum()) == len(set(map(int, idx)))
    s = balancing_strategy(g, "b", engine=eng)
    calls = eng.calls
    assert s.query(0) == ([], 0) and eng.calls == calls
    # one available row: it is picked, and no draw is consumed whatever the branch
    n = len(g["b_ys"])
    keep = int(np.flatnonzero(avail)[0])
    lab = np.setdiff1d(np.arange(n), np.append(g["b_eval"], keep))
    s = balancing_strategy(dict(g, b_labeled=lab), "b", engine=TwinEngine())
    np.random.seed(4)
    before = np.random.get_state()
    idx, cost = s.query(10.0)
    assert [int(i) for i in idx] == [keep] and cost == 1 and _state_equal(before, np.random.get_state())


@pytest.mark.parametrize("tag", ["a", "b"])
def test_sampler_takes_the_per_step_path_beyond_the_limits(bgold, tag):  # noqa: F811
    g = bgold
    eng = TwinEngine(centre_floats=0)
    s = balancing_strategy(g, tag, engine=eng)
    np.random.seed(11)
    idx, cost = s.query(float(g[f"{tag}_budget"]))
    assert eng.declined == 1
    assert [int(i) for i in idx] == g[f"{tag}_picks"].tolist() and cost == int(g[f"{tag}_budget"])
    after = np.random.random_sample()
    _, want = _run_twin(g, tag)
    assert after == want


def test_balancing_desc_layout_matches_header_field_order():
    from active_learning_b200 import _lib
    src = open(os.path.join(ROOT, "include", "alq.h")).read()
    body = src[src.index("typedef struct alq_balancing_desc {"):src.index("} alq_balancing_desc;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = re.findall(r"(\w+)\s*;", body)
    assert fields == [f[0] for f in _lib.BalancingDesc._fields_]
