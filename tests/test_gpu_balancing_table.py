"""K12 (alq_balancing_table_select) on the GPU: BalancingSampler over the incremental row x class table against the
reference's picks, its NumPy twin (tests/balancing_table_oracle.py) and the per-step path, including NumPy's RNG state
after the query, at ImageNet-LT's 1 000 classes."""
import os
import re
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from balancing_table_oracle import balancing_table
from test_balancing import balancing_strategy, bgold, masks  # noqa: F401  (fixture)
from test_balancing_loop import _state_equal, lgold  # noqa: F401  (fixture)
from test_balancing_table import tgold  # noqa: F401  (fixture)
from test_gpu_balancing_loop import imbalanced_counts, make_pool

pytestmark = pytest.mark.gpu

SMEM_CAP = 227 * 1024 - 1024                     # H100's opt-in shared memory per block, less the kernel's static part


@pytest.fixture(scope="module")
def eng():
    from active_learning_b200.engine import Engine
    e = Engine()
    yield e
    e.set_option("balancing_loop", 0)


class option:
    def __init__(self, eng, value):
        self.eng, self.value = eng, value

    def __enter__(self):
        self.eng.set_option("balancing_loop", self.value)

    def __exit__(self, *exc):
        self.eng.set_option("balancing_loop", 0)


def run_table(eng, emb, ys, avail, lab, c, budget, seed):
    """-> (picks, balancing steps, NumPy state after) of K12, or None if it declined."""
    x = torch.from_numpy(np.ascontiguousarray(emb)).cuda()
    np.random.seed(seed)
    res = eng.balancing_table_select(x, eng.row_norm2(x), torch.from_numpy(np.asarray(ys, dtype=np.int32)).cuda(),
                                     torch.from_numpy(avail.astype(np.uint8)).cuda(),
                                     torch.from_numpy(lab.astype(np.uint8)).cuda(), c, budget)
    if res is None:
        return None
    return res[0].tolist(), res[1], np.random.get_state()


def run_twin(emb, ys, avail, lab, c, budget, seed):
    np.random.seed(seed)
    return balancing_table(emb, ys, avail, lab, c, budget)


def pend_cap(c, d, grid=132):
    fixed = 20 * c + 4 * grid + 4 * 624 + 64
    return min(64, (SMEM_CAP - fixed) // (4 * d + 4))


def _golden_case(g, tag):
    avail, lb = masks(g, tag)
    return g[f"{tag}_emb"], g[f"{tag}_ys"], avail, lb, int(g[f"{tag}_classes"]), int(g[f"{tag}_budget"])


@pytest.mark.parametrize("src,tag", [("b", "a"), ("b", "b"), ("l", "m"), ("l", "r"), ("t", "t"), ("t", "u")])
def test_option3_reproduces_every_balancing_golden(eng, bgold, lgold, tgold, src, tag):  # noqa: F811
    g = {"b": bgold, "l": lgold, "t": tgold}[src]
    emb, ys, avail, lb, c, budget = _golden_case(g, tag)
    seed = int(g.get(f"{tag}_seed", 11))
    with option(eng, 3):
        got = run_table(eng, emb, ys, avail, lb, c, budget, seed)
    assert got[0] == g[f"{tag}_picks"].tolist() and got[1] == int(g[f"{tag}_balancing_steps"])
    np.random.set_state(got[2])
    after = np.random.random_sample()
    if f"{tag}_after" in g:
        assert after == float(g[f"{tag}_after"])
    else:
        np.random.set_state(run_twin(emb, ys, avail, lb, c, budget, seed)["state"])
        assert after == np.random.random_sample()


@pytest.mark.parametrize("tag", ["t", "u"])
def test_auto_runs_k12_through_the_sampler(eng, tgold, tag):  # noqa: F811
    g = tgold
    s = balancing_strategy(g, tag, engine=eng)
    np.random.seed(int(g[f"{tag}_seed"]))
    before = eng.launches
    idx, cost = s.query(float(g[f"{tag}_budget"]))
    assert [int(i) for i in idx] == g[f"{tag}_picks"].tolist() and cost == int(g[f"{tag}_budget"])
    assert np.random.random_sample() == float(g[f"{tag}_after"])
    assert eng.launches - before <= 8                    # K11 declined at once, K12 ran: not ~6 launches per pick


def test_imagenet_lt_shape_equals_twin(eng, tgold):  # noqa: F811
    counts = tgold["lt_counts"]
    c, d, budget = 1000, 2048, 200
    rng = np.random.default_rng(7)
    ys = rng.permutation(np.repeat(np.arange(c), counts))
    n = len(ys)
    centres = (rng.standard_normal((c, d), dtype=np.float32) * 0.5)
    emb = centres[ys]
    emb += rng.standard_normal((n, d), dtype=np.float32)
    np.maximum(emb, 0, out=emb)
    lab = np.zeros(n, dtype=bool)
    lab[rng.choice(n, size=n // 10, replace=False)] = True
    avail = ~lab
    checked = 0
    for seed in (1, 2, 3):
        out = run_twin(emb, ys, avail, lab, c, budget, seed)
        if out["min_gap"] < 1e-9:
            continue
        got = run_table(eng, emb, ys, avail, lab, c, budget, seed)
        assert got is not None                           # auto: K12 within its limits
        assert got[0] == out["picks"] and got[1] == out["balancing_steps"] and _state_equal(got[2], out["state"])
        assert out["balancing_steps"] == budget
        checked += 1
        break
    assert checked == 1


def test_per_step_path_equals_auto_at_1000_classes(eng):
    n, d, c, budget = 20431, 512, 1000, 40
    from helpers import LabeledIndexDataset, make_strategy
    checked = 0
    for seed in range(6):
        if checked == 2:
            break
        emb, ys, avail, lab = make_pool(n, d, c, seed, imbalanced_counts(c, 12, 0.1))
        out = run_twin(emb, ys, avail, lab, c, budget, seed)
        if out["min_gap"] < 1e-4:
            continue
        picks = {}
        for opt in (0, 1):
            s = make_strategy("BalancingSampler", torch.zeros(n, c), torch.from_numpy(emb), np.zeros(0, dtype=np.int64),
                              np.flatnonzero(lab), 1024, engine=eng, dataset=LabeledIndexDataset(ys, c))
            with option(eng, opt):
                np.random.seed(seed)
                idx, _ = s.query(float(budget))
            picks[opt] = ([int(i) for i in idx], np.random.get_state())
        assert picks[0][0] == picks[1][0] == out["picks"] and _state_equal(picks[0][1], picks[1][1])
        checked += 1
    assert checked >= 1


def test_edges(eng):
    from active_learning_b200.engine import AlqError
    n, d, c = 3000, 24, 1000
    emb, ys, avail, lab = make_pool(n, d, c, 5, [2] * 500 + [0] * 500)      # half the classes have no labeled row
    with option(eng, 3):
        out = run_twin(emb, ys, avail, lab, c, 25, 2)
        got = run_table(eng, emb, ys, avail, lab, c, 25, 2)
        assert got[0] == out["picks"] and got[1] == out["balancing_steps"] and _state_equal(got[2], out["state"])
        # budget 0 and 1, and larger than the available rows
        np.random.seed(8)
        before = np.random.get_state()
        assert run_table(eng, emb, ys, avail, lab, c, 0, 8)[:2] == ([], 0)
        np.random.seed(8)
        assert _state_equal(before, np.random.get_state())
        assert run_table(eng, emb, ys, avail, lab, c, 1, 2)[0] == run_twin(emb, ys, avail, lab, c, 1, 2)["picks"]
        small = avail.copy()
        small[np.flatnonzero(small)[30:]] = False
        out = run_twin(emb, ys, small, lab, c, 100, 2)
        got = run_table(eng, emb, ys, small, lab, c, 100, 2)
        assert len(got[0]) == 30 and sorted(got[0]) == np.flatnonzero(small).tolist() and got[0] == out["picks"]
        # one available row
        one = np.zeros(n, dtype=bool)
        one[1234] = True
        np.random.seed(3)
        before = np.random.get_state()
        got = run_table(eng, emb, ys, one, lab & ~one, c, 10, 3)
        assert got[0] == [1234] and _state_equal(before, got[2])
        # duplicated rows: every ratio ties, the lowest row wins
        dup = emb.copy()
        dup[avail] = dup[np.flatnonzero(avail)[0]]
        got = run_table(eng, dup, ys, avail, lab, c, 40, 1)
        assert got[1] == 40 and got[0] == np.flatnonzero(avail)[:40].tolist()
        # out-of-range labels, before any draw
        bad = ys.copy()
        row = int(np.flatnonzero(avail)[17])
        bad[row] = c
        np.random.seed(8)
        with pytest.raises(AlqError, match=f"available row {row} has label {c}"):
            run_table(eng, emb, bad, avail, lab, c, 10, 8)
        after = np.random.get_state()
        assert _state_equal(after, _seeded_state(8))
        bad = ys.copy()
        row = int(np.flatnonzero(lab)[3])
        bad[row] = -2
        with pytest.raises(AlqError, match=f"labeled row {row} has label -2"):
            run_table(eng, emb, bad, avail, lab, c, 10, 8)


def _seeded_state(seed):
    np.random.seed(seed)
    return np.random.get_state()


def test_query_that_never_balances(eng):
    n, budget = 200000, 1500
    rng = np.random.default_rng(1)
    emb = rng.random((n, 8), dtype=np.float32)
    ys = np.zeros(n, dtype=np.int64)                    # one class: every step draws
    lab = np.zeros(n, dtype=bool)
    lab[rng.choice(n, size=2000, replace=False)] = True
    with option(eng, 3):
        got = run_table(eng, emb, ys, ~lab, lab, 1, budget, 5)
    out = run_twin(emb, ys, ~lab, lab, 1, budget, 5)
    assert got[1] == 0 and got[0] == out["picks"] and _state_equal(got[2], out["state"]) and out["table"] is None


def test_random_run_longer_than_the_pending_list(eng, tgold):  # noqa: F811
    """The uniform C = 1 000 golden with every embedding tiled 341 times (16 368 dimensions; distances scale, ratios do
    not): the pending list holds 3 rows there, and after its first balancing step the query draws runs of up to 12
    random rows, so the CTAs flush the list on their own."""
    g = tgold
    emb, ys, avail, lb, c, budget = _golden_case(g, "u")
    big = np.ascontiguousarray(np.tile(emb, (1, 341)))
    cap = pend_cap(c, big.shape[1])
    out = run_twin(emb, ys, avail, lb, c, budget, int(g["u_seed"]))
    br = out["branch"]
    runs, cur = [], 0
    for b in br[br.index(True):]:
        cur = 0 if b else cur + 1
        runs.append(cur)
    assert 1 <= cap < max(runs)
    with option(eng, 3):
        got = run_table(eng, big, ys, avail, lb, c, budget, int(g["u_seed"]))
    assert got[0] == g["u_picks"].tolist() and got[1] == int(g["u_balancing_steps"])
    np.random.set_state(got[2])
    assert np.random.random_sample() == float(g["u_after"])


def test_limits(eng):
    from active_learning_b200.engine import AlqError
    # per-class tables in shared memory: 12 000 classes need 240 000 bytes
    emb, ys, avail, lab = make_pool(2000, 4, 12000, 1, [0] * 12000)
    assert run_table(eng, emb, ys, avail, lab, 12000, 10, 1) is None
    with option(eng, 3), pytest.raises(AlqError, match="class tables in shared memory"):
        run_table(eng, emb, ys, avail, lab, 12000, 10, 1)
    # rows per CTA segment: more than 65 535 rows per CTA
    n = 65536 * torch.cuda.get_device_properties(0).multi_processor_count + 1000
    emb = np.zeros((n, 4), dtype=np.float32)
    ys = np.zeros(n, dtype=np.int64)
    lab = np.zeros(n, dtype=bool)
    lab[:10] = True
    assert run_table(eng, emb, ys, ~lab, lab, 2, 10, 1) is None
    with option(eng, 3), pytest.raises(AlqError, match="rows per segment"):
        run_table(eng, emb, ys, ~lab, lab, 2, 10, 1)
    del emb
    # the table in device memory: 1.4 M available rows x 8 000 classes = 89.6 GB; found out without reserving it
    n, c = 1400000, 8000
    emb = np.random.default_rng(0).random((n, 4), dtype=np.float32)
    ys = np.arange(n, dtype=np.int64) % c
    lab = np.zeros(n, dtype=bool)
    lab[:c] = True
    run_table(eng, emb[:1000], ys[:1000], ~lab[:1000], lab[:1000], c, 0, 1)   # warm the allocator and the library
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    assert run_table(eng, emb, ys, ~lab, lab, c, 10, 1) is None
    with option(eng, 3), pytest.raises(AlqError, match="table in device memory"):
        run_table(eng, emb, ys, ~lab, lab, c, 10, 1)
    torch.cuda.synchronize()
    assert free0 - torch.cuda.mem_get_info()[0] < (1 << 30)
    # options 1 and 2 decline; option 3 makes K11 decline
    emb, ys, avail, lab = make_pool(2000, 64, 10, 1, [5] * 10)
    for opt in (1, 2):
        with option(eng, opt):
            assert run_table(eng, emb, ys, avail, lab, 10, 10, 1) is None
    x = torch.from_numpy(emb).cuda()
    with option(eng, 3):
        assert eng.balancing_select(x, eng.row_norm2(x), torch.from_numpy(ys.astype(np.int32)).cuda(),
                                    torch.from_numpy(avail.astype(np.uint8)).cuda(),
                                    torch.from_numpy(lab.astype(np.uint8)).cuda(), 10, 10) is None


def test_two_runs_are_bitwise_identical(eng):
    emb, ys, avail, lab = make_pool(20431, 512, 1000, 21, imbalanced_counts(1000, 10))
    a = run_table(eng, emb, ys, avail, lab, 1000, 100, 6)
    b = run_table(eng, emb, ys, avail, lab, 1000, 100, 6)
    assert a[0] == b[0] and a[1] == b[1] and _state_equal(a[2], b[2])


def test_launch_count_does_not_depend_on_the_budget(eng):
    emb, ys, avail, lab = make_pool(20431, 64, 1000, 2, imbalanced_counts(1000, 10))
    counts = []
    for budget in (10, 800):
        before = eng.launches
        got = run_table(eng, emb, ys, avail, lab, 1000, budget, 1)
        counts.append(eng.launches - before)
        assert len(got[0]) == budget
    assert counts[0] == counts[1] <= 8


def test_k12_compiles_without_spills():
    """ptxas's register and spill report of K12's three kernels for sm_90a."""
    import shutil
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    src = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "active_learning_b200", "csrc",
                       "alq_balancing_table.cu")
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                            "-c", src, "-o", os.path.join(tmp, "k12.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    report = re.findall(r"Compiling entry function '(\w*(?:bal_|balancing_)\w*kernel\w*)'.*?(\d+) bytes spill stores, (\d+) "
                        r"bytes spill loads.*?Used (\d+) registers", r.stderr, flags=re.S)
    assert len(report) == 3
    for name, stores, loads, regs in report:
        print(f"{name}: {regs} registers, spills {stores} B stored / {loads} B loaded", file=sys.stderr)
        assert stores == loads == "0"
