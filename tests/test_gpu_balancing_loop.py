"""K11 (alq_balancing_select) on the GPU: the persistent BalancingSampler loop against the reference's picks, its NumPy
twin (tests/balancing_loop_oracle.py) and the per-step path, including NumPy's RNG state after the query."""
import os
import re
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from balancing_loop_oracle import balancing_loop
from test_balancing import balancing_strategy, bgold, masks  # noqa: F401  (fixture)
from test_balancing_loop import _state_equal, lgold  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from active_learning_b200.engine import Engine
    e = Engine()
    yield e
    e.set_option("balancing_loop", 0)


def make_pool(n, d, c, seed, lab_counts, scale=2.0):
    """Rows relu(centre of the row's class + noise); lab_counts[k] labeled rows of class k; every other row available."""
    rng = np.random.default_rng(seed)
    ys = rng.integers(0, c, size=n)
    centres = rng.normal(size=(c, d)) * scale
    emb = np.maximum(centres[ys] + rng.normal(size=(n, d)), 0).astype(np.float32)
    lab = np.zeros(n, dtype=bool)
    for k in range(c):
        rows = np.flatnonzero(ys == k)
        lab[rng.choice(rows, size=min(len(rows), int(lab_counts[k])), replace=False)] = True
    return emb, ys, ~lab, lab


def run_loop(eng, emb, ys, avail, lab, c, budget, seed):
    """-> (picks, balancing steps, NumPy state after) of the device loop, or None if it declined."""
    x = torch.from_numpy(emb).cuda()
    np.random.seed(seed)
    res = eng.balancing_select(x, eng.row_norm2(x), torch.from_numpy(np.asarray(ys, dtype=np.int32)).cuda(),
                               torch.from_numpy(avail.astype(np.uint8)).cuda(), torch.from_numpy(lab.astype(np.uint8)).cuda(),
                               c, budget)
    if res is None:
        return None
    return res[0].tolist(), res[1], np.random.get_state()


def run_twin(emb, ys, avail, lab, c, budget, seed):
    np.random.seed(seed)
    return balancing_loop(emb, ys, avail, lab, c, budget)


def imbalanced_counts(c, top, factor=0.1):
    """CIFAR-LT style: class k keeps top * factor^(k / (c - 1)) labeled rows."""
    return [max(1, int(top * factor ** (k / max(c - 1, 1)))) for k in range(c)]


@pytest.mark.parametrize("tag", ["a", "b"])
def test_sampler_returns_the_balancing_goldens(eng, bgold, tag):  # noqa: F811
    g = bgold
    s = balancing_strategy(g, tag, engine=eng)
    np.random.seed(11)
    launches = eng.launches
    idx, cost = s.query(float(g[f"{tag}_budget"]))
    assert [int(i) for i in idx] == g[f"{tag}_picks"].tolist() and cost == int(g[f"{tag}_budget"])
    assert eng.launches - launches <= 8                 # the loop ran: a handful of launches, not ~15 per pick
    after = np.random.random_sample()
    avail, lb = masks(g, tag)
    out = run_twin(g[f"{tag}_emb"], g[f"{tag}_ys"], avail, lb, int(g[f"{tag}_classes"]), int(g[f"{tag}_budget"]), 11)
    np.random.set_state(out["state"])
    assert after == np.random.random_sample()           # equal to the reference's (tests/test_balancing.py)


@pytest.mark.parametrize("tag", ["m", "r"])
def test_sampler_returns_the_loop_goldens(eng, lgold, tag):  # noqa: F811
    g = lgold
    s = balancing_strategy(g, tag, engine=eng)
    np.random.seed(int(g[f"{tag}_seed"]))
    idx, cost = s.query(float(g[f"{tag}_budget"]))
    assert [int(i) for i in idx] == g[f"{tag}_picks"].tolist() and cost == int(g[f"{tag}_budget"])
    assert np.random.random_sample() == float(g[f"{tag}_after"])
    assert s._bal_cache[0].is_cuda


def test_random_only_at_imagenet_size(eng):
    n, budget = 1281167, 2000
    rng = np.random.default_rng(1)
    emb = rng.random((n, 4), dtype=np.float32)
    ys = np.zeros(n, dtype=np.int64)                    # one class: every step draws
    lab = np.zeros(n, dtype=bool)
    lab[rng.choice(n, size=12000, replace=False)] = True
    got = run_loop(eng, emb, ys, ~lab, lab, 1, budget, 5)
    out = run_twin(emb, ys, ~lab, lab, 1, budget, 5)
    assert got[1] == 0 and got[0] == out["picks"]
    assert _state_equal(got[2], out["state"]) and out["outputs"] > budget   # the same MT outputs consumed


@pytest.mark.parametrize("kind", ["mixed", "balancing"])
def test_cifar_shape_loop_equals_per_step_path_and_twin(eng, kind):
    n, d, c = 20431, 512, 10
    from helpers import LabeledIndexDataset, make_strategy
    checked = 0
    for seed in range(6):                                # seeds whose twin gap is >= 1e-4: 0-2 mixed, 3 balancing
        if checked == 2:
            break
        if kind == "mixed":                              # a near-balanced labeled set: random first, balancing at the end
            emb, ys, avail, lab = make_pool(n, d, c, seed, [100] * 9 + [97])
            budget = 120
        else:                                            # CIFAR-10-LT's exp factor 0.1 over 1000 labeled rows
            emb, ys, avail, lab = make_pool(n, d, c, seed, imbalanced_counts(c, 400))
            budget = 50
        out = run_twin(emb, ys, avail, lab, c, budget, seed)
        if out["min_gap"] < 1e-4:
            continue
        got = run_loop(eng, emb, ys, avail, lab, c, budget, seed)
        assert got[0] == out["picks"] and got[1] == out["balancing_steps"] and _state_equal(got[2], out["state"])
        if kind == "balancing":
            assert out["balancing_steps"] == budget
        else:
            assert 0 < out["balancing_steps"] < budget
        # the per-step path through the sampler (option balancing_loop = 1) makes the same picks
        s = make_strategy("BalancingSampler", torch.zeros(n, c), torch.from_numpy(emb), np.zeros(0, dtype=np.int64),
                          np.flatnonzero(lab), 1024, engine=eng, dataset=LabeledIndexDataset(ys, c))
        eng.set_option("balancing_loop", 1)
        try:
            np.random.seed(seed)
            idx, cost = s.query(float(budget))
        finally:
            eng.set_option("balancing_loop", 0)
        assert [int(i) for i in idx] == out["picks"] and _state_equal(np.random.get_state(), out["state"])
        checked += 1
    assert checked >= 1


@pytest.mark.parametrize("n", [1023, 1024, 1025, 16895, 16896, 16897, 20000])
def test_segment_edges(eng, n):
    c, d = 5, 32
    emb, ys, avail, lab = make_pool(n, d, c, n, [40, 20, 10, 5, 0])
    for budget in (60, n):                               # balancing, then all rows (random steps mixed in)
        budget = min(budget, 400)
        out = run_twin(emb, ys, avail, lab, c, budget, 3)
        if out["min_gap"] < 1e-4:
            continue
        got = run_loop(eng, emb, ys, avail, lab, c, budget, 3)
        assert got[0] == out["picks"] and got[1] == out["balancing_steps"] and _state_equal(got[2], out["state"])


def test_duplicated_rows_lowest_row_wins(eng):
    n, d, c = 5000, 16, 4
    emb, ys, avail, lab = make_pool(n, d, c, 9, [50, 20, 5, 0])
    emb[avail] = emb[np.flatnonzero(avail)[0]]           # every available row is the same row: every ratio ties
    got = run_loop(eng, emb, ys, avail, lab, c, 40, 1)
    assert got[1] == 40 and got[0] == np.flatnonzero(avail)[:40].tolist()


def test_numerator_one_branch_budget_edges_and_bad_label(eng):
    from active_learning_b200.engine import AlqError
    n, d, c = 3000, 24, 6
    emb, ys, avail, lab = make_pool(n, d, c, 5, [60, 30, 15, 8, 4, 0])   # the rarest class has no labeled row
    out = run_twin(emb, ys, avail, lab, c, 25, 2)
    got = run_loop(eng, emb, ys, avail, lab, c, 25, 2)
    assert out["min_gap"] >= 1e-4 and got[0] == out["picks"] and got[1] == 25
    small = avail.copy()
    small[np.flatnonzero(small)[30:]] = False           # 30 available rows, budget 100: all of them
    out = run_twin(emb, ys, small, lab, c, 100, 2)
    got = run_loop(eng, emb, ys, small, lab, c, 100, 2)
    assert len(got[0]) == 30 and sorted(got[0]) == np.flatnonzero(small).tolist() and got[0] == out["picks"]
    np.random.seed(8)
    before = np.random.get_state()
    assert run_loop(eng, emb, ys, avail, lab, c, 0, 8)[:2] == ([], 0)
    np.random.seed(8)
    assert _state_equal(before, np.random.get_state())
    bad = ys.copy()
    row = int(np.flatnonzero(avail)[17])
    bad[row] = c
    np.random.seed(8)
    with pytest.raises(AlqError, match=f"available row {row} has label {c}"):
        run_loop(eng, emb, bad, avail, lab, c, 10, 8)
    assert _state_equal(before, np.random.get_state())  # rejected before any draw
    bad = ys.copy()
    row = int(np.flatnonzero(lab)[3])
    bad[row] = -2
    with pytest.raises(AlqError, match=f"labeled row {row} has label -2"):
        run_loop(eng, emb, bad, avail, lab, c, 10, 8)


def test_two_runs_are_bitwise_identical(eng):
    emb, ys, avail, lab = make_pool(20431, 512, 10, 21, imbalanced_counts(10, 300))
    a = run_loop(eng, emb, ys, avail, lab, 10, 200, 6)
    b = run_loop(eng, emb, ys, avail, lab, 10, 200, 6)
    assert a[0] == b[0] and a[1] == b[1] and _state_equal(a[2], b[2])


def test_limits_and_auto_fallback(eng):
    from active_learning_b200.engine import AlqError
    emb, ys, avail, lab = make_pool(2000, 512, 1000, 1, [1] * 1000)   # 1000 centres of 512 floats: 2 MB
    assert run_loop(eng, emb, ys, avail, lab, 1000, 10, 1) is None       # auto: the per-step path runs
    eng.set_option("balancing_loop", 2)
    try:
        with pytest.raises(AlqError, match="centres in shared memory"):
            run_loop(eng, emb, ys, avail, lab, 1000, 10, 1)
    finally:
        eng.set_option("balancing_loop", 0)
    emb, ys, avail, lab = make_pool(2000, 2048, 10, 1, [5] * 10)          # C = 10, D = 2048 fits
    assert run_loop(eng, emb, ys, avail, lab, 10, 10, 1) is not None
    eng.set_option("balancing_loop", 1)
    try:
        assert run_loop(eng, emb, ys, avail, lab, 10, 10, 1) is None
    finally:
        eng.set_option("balancing_loop", 0)


def test_launch_count_does_not_depend_on_the_budget(eng):
    emb, ys, avail, lab = make_pool(20431, 64, 10, 2, imbalanced_counts(10, 300))
    counts = []
    for budget in (10, 800):
        before = eng.launches
        got = run_loop(eng, emb, ys, avail, lab, 10, budget, 1)
        counts.append(eng.launches - before)
        assert len(got[0]) == budget
    assert counts[0] == counts[1] <= 8


def test_k11_compiles_without_spills():
    """ptxas's register and spill report of K11's four kernels for sm_90a."""
    import shutil
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    src = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "active_learning_b200", "csrc",
                       "alq_balancing.cu")
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                            "-c", src, "-o", os.path.join(tmp, "k11.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    report = re.findall(r"Compiling entry function '(\w*(?:bal_|balancing_)\w*kernel\w*)'.*?(\d+) bytes spill stores, (\d+) "
                        r"bytes spill loads.*?Used (\d+) registers", r.stderr, flags=re.S)
    assert len(report) == 4
    for name, stores, loads, regs in report:
        print(f"{name}: {regs} registers, spills {stores} B stored / {loads} B loaded", file=sys.stderr)
        assert stores == loads == "0"
