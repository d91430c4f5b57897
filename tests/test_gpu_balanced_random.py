"""K10 / BalancedRandomSampler on the H100: class counts against np.bincount across tile edges and class counts up to
the shared-memory bound, argument checks, the picks against NumPy's nonzero + permutation, the whole query on the
reference's goldens (picks and torch RNG state), and an ImageNet-sized pool against the oracle with a launch count
that does not grow with the number of classes."""
import ctypes
import os
import re
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

import balanced_random_oracle as BR

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
CLASS_MAX, TILE = 32768, 1024


@pytest.fixture(scope="module")
def eng():
    from active_learning_b200.engine import Engine
    return Engine()


def tile_of(c):
    return TILE * ((c + TILE - 1) // TILE)


def pool(n, c, seed, p_avail=0.7):
    rng = np.random.default_rng(seed)
    ys = rng.integers(0, c, n).astype(np.int32)
    av = rng.random(n) < p_avail
    # unavailable rows may carry any label: the kernels never look at them
    junk = ~av & (rng.random(n) < 0.2)
    ys[junk] = rng.choice(np.array([-7, c, c + 100, 2 ** 31 - 1], dtype=np.int64), junk.sum()).astype(np.int32)
    return ys, av


def dev(ys, av):
    return torch.from_numpy(ys).cuda(), torch.from_numpy(av.astype(np.uint8)).cuda()


@pytest.mark.parametrize("c", [1, 10, 1000, CLASS_MAX])
def test_counts_equal_bincount(eng, c):
    t = tile_of(c)
    for n in sorted({1, 31, t - 1, t, t + 1, 1281167}):
        ys, av = pool(n, c, n + c)
        counts = eng.class_counts(*dev(ys, av), c).cpu().numpy()
        assert np.array_equal(counts, np.bincount(ys[av], minlength=c)), (n, c)


def test_invalid_arguments_are_rejected(eng):
    from active_learning_b200._lib import AlqError
    lib, st = eng.lib, eng._stream()
    ys, av = pool(5000, 10, 1)
    labels, avail = dev(ys, av)
    counts = torch.empty(CLASS_MAX + 1, dtype=torch.int32, device="cuda")
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731

    def cnt(n=5000, c=10, lp=None, ap=None, cp=None):
        return lib.alq_class_counts(eng._h, lp if lp is not None else P(labels), ap if ap is not None else P(avail), n, c,
                                    cp if cp is not None else P(counts), st)

    assert cnt() == 0
    for kw in (dict(c=CLASS_MAX + 1), dict(c=0), dict(n=-1), dict(n=2 ** 31), dict(lp=ctypes.c_void_p(0)),
               dict(ap=ctypes.c_void_p(0)), dict(cp=ctypes.c_void_p(0))):
        assert cnt(**kw) == 1, kw                          # ALQ_ERR_INVALID
    # a bad label on an available row: invalid, and the message names the smallest such row and its label
    bad = ys.copy()
    i = int(np.flatnonzero(av)[100])
    bad[i], bad[int(np.flatnonzero(av)[200])] = 10, -3
    with pytest.raises(AlqError, match=f"row {i} has label 10"):
        eng.class_counts(torch.from_numpy(bad).cuda(), avail, 10)
    # ... and ignored on an unavailable row
    j = int(np.flatnonzero(~av)[0])
    bad = ys.copy()
    bad[j] = 99
    assert np.array_equal(eng.class_counts(torch.from_numpy(bad).cuda(), avail, 10).cpu().numpy(),
                          np.bincount(ys[av], minlength=10))
    k = torch.zeros(10, dtype=torch.int32, device="cuda")
    out = torch.empty(4, dtype=torch.int32, device="cuda")

    def pick(n=5000, c=10, b=4, kp=None, pp=None, op=None):
        return lib.alq_class_pick(eng._h, P(labels), P(avail), n, c, kp if kp is not None else P(k),
                                  pp if pp is not None else P(k), b, op if op is not None else P(out), st)

    for kw in (dict(c=CLASS_MAX + 1), dict(c=0), dict(b=-1), dict(n=-1), dict(kp=ctypes.c_void_p(0)),
               dict(pp=ctypes.c_void_p(0)), dict(op=ctypes.c_void_p(0))):
        assert pick(**kw) == 1, kw
    for args in ((labels.cpu(), avail), (labels, avail[:10]), (labels.long(), avail)):
        with pytest.raises(AlqError):
            eng.class_counts(*args, 10)
    with pytest.raises(AlqError):
        eng.class_counts(labels, avail, CLASS_MAX + 1)
    with pytest.raises(AlqError):
        eng.class_pick(labels, avail, [1, 2], [0, 0])       # sum(k) != len(perm)
    with pytest.raises(AlqError):
        eng.class_pick(labels, avail, [1, -1], [0])
    torch.cuda.synchronize()


def reference_pick(ys, av, k, perm):
    out, at = [], 0
    for c in range(len(k)):
        rows = np.flatnonzero((ys == c) & av)
        out += [int(rows[r]) if r < len(rows) else -1 for r in perm[at:at + k[c]]]
        at += k[c]
    return out


@pytest.mark.parametrize("c", [1, 10, 1000, 5000])
def test_pick_equals_nonzero_of_the_permutation(eng, c):
    t = tile_of(c)
    n = 7 * t + 123
    ys, av = pool(n, c, 3 * c)
    # class c - 1 lives only on tile edges: rows t*q - 1 and t*q
    edge = np.array([r for q in range(1, 7) for r in (t * q - 1, t * q)])
    if c > 1:
        ys[ys == c - 1] = 0
    ys[edge], av[edge] = c - 1, True
    counts = np.bincount(ys[av], minlength=c)
    rng = np.random.default_rng(c)
    k = np.where(rng.random(c) < 0.3, 0, rng.integers(0, counts + 1))    # some classes take nothing
    k[c - 1] = counts[c - 1]
    perms = []
    for cls in range(c):
        full = rng.permutation(counts[cls])
        if k[cls] >= 2:                                                    # first and last available row of the class
            last = counts[cls] - 1
            full = np.concatenate([[0, last], full[(full != 0) & (full != last)]])
        perms.append(full[:k[cls]])
    perm = np.concatenate(perms).astype(np.int64)
    labels, avail = dev(ys, av)
    got = eng.class_pick(labels, avail, k, perm).cpu().numpy().tolist()
    assert got == reference_pick(ys, av, k, perm)
    assert set(edge.tolist()) <= set(got)
    # ranks at or past a class's count give -1 (raw call: the engine only checks the sizes)
    bad = perm.copy()
    cls = int(np.flatnonzero(k > 0)[0])
    bad[int(k[:cls].sum())] = counts[cls]
    got = eng.class_pick(labels, avail, k, bad).cpu().numpy()
    assert got[int(k[:cls].sum())] == -1 and got.tolist() == reference_pick(ys, av, k, bad)


@pytest.mark.parametrize("tag", ["balanced", "longtail", "all", "c1000", "zero", "ties"])
def test_query_replays_the_reference_goldens(eng, tag):
    from test_balanced_random import assert_golden, fixture_sampler, golden_query, load_gold, skip_unusable
    gold = load_gold()
    skip_unusable(gold, tag)
    s = fixture_sampler(gold, tag, eng)
    assert_golden(gold, tag, *golden_query(gold, s, tag))


def test_imagenet_scale_equals_the_oracle_with_a_constant_launch_count(eng):
    from test_balanced_random import make_sampler
    n, budget = 1281167, 10000.0
    deltas = {}
    for c in (10, 1000):
        rng = np.random.default_rng(c)
        ys = rng.integers(0, c, n)
        ev = rng.choice(n, 12000, replace=False)
        s = make_sampler(ys, c, ev, [], eng)
        torch.manual_seed(0)
        before = eng.launches
        idx, cost = s.query(budget)
        deltas[c] = eng.launches - before
        d = BR.torch_rng_digest()
        torch.manual_seed(0)
        oidx, ocost = BR.balanced_random_query(ys.tolist(), s.available_query_idxs(boolean=True), c, budget)
        assert (idx, cost) == (oidx, ocost) and BR.torch_rng_digest() == d
    assert deltas[10] == deltas[1000] <= 8, deltas


def test_k10_compiles_without_spills():
    """ptxas's register and spill report of K10 for sm_90a."""
    import shutil
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    src = os.path.join(os.path.dirname(HERE), "active_learning_b200", "csrc", "alq_classes.cu")
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                            "-c", src, "-o", os.path.join(tmp, "k10.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    report = re.findall(r"Compiling entry function '(\w*class_\w*kernel\w*)'.*?(\d+) bytes spill stores, (\d+) bytes spill "
                        r"loads.*?Used (\d+) registers", r.stderr, flags=re.S)
    assert len(report) == 4
    for name, stores, loads, regs in report:
        print(f"{name}: {regs} registers, spills {stores} B stored / {loads} B loaded", file=sys.stderr)
        assert stores == loads == "0"
