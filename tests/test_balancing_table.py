"""K12, BalancingSampler over the incremental row x class table, on the CPU: its NumPy twin
(tests/balancing_table_oracle.py) against the picks the reference itself produced at C = 1 000 and on the K11 goldens,
the incremental table against a fresh fp64 evaluation, and the sampler's routing K11 -> K12 -> per-step path."""
import os

import numpy as np
import pytest

from balancing_table_oracle import balancing_table
from test_balancing import balancing_strategy, bgold, masks  # noqa: F401  (fixture)
from test_balancing_loop import TwinEngine, _state_equal, lgold  # noqa: F401  (fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def tgold():
    return dict(np.load(os.path.join(ROOT, "tests", "golden", "reference_golden_balancing_table.npz")))


def _run_twin(g, tag):
    avail, lb = masks(g, tag)
    np.random.seed(int(g.get(f"{tag}_seed", 11)))
    out = balancing_table(g[f"{tag}_emb"], g[f"{tag}_ys"], avail, lb, int(g[f"{tag}_classes"]), int(g[f"{tag}_budget"]))
    np.random.set_state(out["state"])
    return out, np.random.random_sample()


def test_lt_profile_is_imagenet_lt(tgold):
    counts = tgold["lt_counts"]
    assert len(counts) == 1000 and counts.sum() == 115846 and counts.min() == 5 and counts.max() == 1280
    assert int(np.median(counts)) in (72, 73, 74)


@pytest.mark.parametrize("tag", ["t", "u"])
def test_twin_matches_reference_at_1000_classes(tgold, tag):
    g = tgold
    out, after = _run_twin(g, tag)
    assert out["picks"] == g[f"{tag}_picks"].tolist() and after == float(g[f"{tag}_after"])
    assert out["balancing_steps"] == int(g[f"{tag}_balancing_steps"]) and out["min_gap"] >= 1e-4
    avail, lb = masks(g, tag)
    if tag == "t":                                  # every step balances, some rarest classes start with no labeled row
        assert out["balancing_steps"] == int(g["t_budget"])
        assert np.bincount(g["t_ys"][lb], minlength=1000).min() == 0
    else:                                           # random draws first, then balancing
        assert not out["branch"][0] and 0 < out["balancing_steps"] < int(g["u_budget"])


@pytest.mark.parametrize("tag", ["a", "b"])
def test_twin_matches_reference_on_balancing_goldens(bgold, tag):  # noqa: F811
    out, after = _run_twin(bgold, tag)
    assert out["picks"] == bgold[f"{tag}_picks"].tolist()
    assert out["balancing_steps"] == int(bgold[f"{tag}_balancing_steps"])
    _, want = _run_loop_twin(bgold, tag)
    assert after == want


def _run_loop_twin(g, tag):
    from balancing_loop_oracle import balancing_loop
    avail, lb = masks(g, tag)
    np.random.seed(int(g.get(f"{tag}_seed", 11)))
    out = balancing_loop(g[f"{tag}_emb"], g[f"{tag}_ys"], avail, lb, int(g[f"{tag}_classes"]), int(g[f"{tag}_budget"]))
    np.random.set_state(out["state"])
    return out, np.random.random_sample()


@pytest.mark.parametrize("tag", ["m", "r"])
def test_twin_matches_reference_on_loop_goldens(lgold, tag):
    out, after = _run_twin(lgold, tag)
    assert out["picks"] == lgold[f"{tag}_picks"].tolist() and after == float(lgold[f"{tag}_after"])
    assert out["balancing_steps"] == int(lgold[f"{tag}_balancing_steps"])


@pytest.mark.parametrize("tag", ["t", "u"])
def test_incremental_table_equals_fresh_evaluation(tgold, tag):
    g = tgold
    out, _ = _run_twin(g, tag)
    slots = out["slots"]
    fresh = g[f"{tag}_emb"][slots].astype(np.float64) @ out["sums"].T
    scale = np.abs(g[f"{tag}_emb"][slots].astype(np.float64)) @ np.abs(out["sums"]).T
    assert np.all(np.abs(out["table"] - fresh) <= 1e-12 * np.maximum(scale, 1e-300))


def test_twin_rejects_out_of_range_labels(tgold):
    g = tgold
    avail, lb = masks(g, "u")
    ys = g["u_ys"].copy()
    row = int(np.flatnonzero(avail)[5])
    ys[row] = 1000
    with pytest.raises(ValueError, match=f"available row {row} has label 1000"):
        balancing_table(g["u_emb"], ys, avail, lb, 1000, 5)


class TableEngine(TwinEngine):
    """TwinEngine whose K11 declines (C * D beyond `centre_floats`) and whose K12 is the table twin, declining when
    `table_ok` is False."""

    def __init__(self, centre_floats=0, table_ok=True):
        super().__init__(centre_floats)
        self.table_ok = table_ok
        self.table_calls = self.table_declined = 0

    def balancing_table_select(self, emb, xn, labels, avail, labeled, num_classes, budget):
        self.table_calls += 1
        if not self.table_ok:
            self.table_declined += 1
            return None
        out = balancing_table(emb.numpy(), labels.numpy(), avail.numpy().astype(bool), labeled.numpy().astype(bool),
                              num_classes, budget, np.random.get_state())
        np.random.set_state(out["state"])
        return np.asarray(out["picks"], dtype=np.int64), out["balancing_steps"]


@pytest.mark.parametrize("tag", ["t", "u"])
def test_sampler_calls_k12_when_k11_declines(tgold, tag):
    g = tgold
    eng = TableEngine()
    s = balancing_strategy(g, tag, engine=eng)
    np.random.seed(int(g[f"{tag}_seed"]))
    idx, cost = s.query(float(g[f"{tag}_budget"]))
    assert eng.calls == eng.declined == 1 and eng.table_calls == 1 and eng.table_declined == 0
    assert [int(i) for i in idx] == g[f"{tag}_picks"].tolist() and cost == int(g[f"{tag}_budget"])
    assert np.random.random_sample() == float(g[f"{tag}_after"])


@pytest.mark.parametrize("tag", ["a", "b"])
def test_sampler_per_step_path_when_both_decline(bgold, tag):  # noqa: F811
    g = bgold
    eng = TableEngine(table_ok=False)
    s = balancing_strategy(g, tag, engine=eng)
    np.random.seed(11)
    idx, cost = s.query(float(g[f"{tag}_budget"]))
    assert eng.declined == 1 and eng.table_declined == 1
    assert [int(i) for i in idx] == g[f"{tag}_picks"].tolist() and cost == int(g[f"{tag}_budget"])
    after = np.random.random_sample()
    _, want = _run_loop_twin(g, tag)
    assert after == want


def test_sampler_without_k12_behaves_as_before(bgold):  # noqa: F811
    g = bgold
    eng = TwinEngine(centre_floats=0)               # K11 declines and there is no balancing_table_select
    assert not hasattr(eng, "balancing_table_select")
    s = balancing_strategy(g, "a", engine=eng)
    np.random.seed(11)
    idx, _ = s.query(float(g["a_budget"]))
    assert eng.declined == 1 and [int(i) for i in idx] == g["a_picks"].tolist()
    eng = TableEngine(centre_floats=1 << 20)        # K11 runs: K12 is never asked
    s = balancing_strategy(g, "a", engine=eng)
    np.random.seed(11)
    idx, _ = s.query(float(g["a_budget"]))
    assert eng.calls == 1 and eng.table_calls == 0 and [int(i) for i in idx] == g["a_picks"].tolist()


def test_table_entry_point_is_bound():
    from active_learning_b200 import _lib
    assert _lib.ABI_VERSION == 10 and "alq_balancing_table_select" in _lib.SIGNATURES
    src = open(os.path.join(ROOT, "include", "alq.h")).read()
    assert "int alq_balancing_table_select(alq_ctx* ctx, const alq_balancing_desc* desc, void* stream);" in src
