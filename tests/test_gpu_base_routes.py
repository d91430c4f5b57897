"""BASE's selection (alq_base_select, csrc/alq_mase.cu) on every route and at the branches random pools never reach:
forced fail flags, lists that run out, ties, +inf keys, the route boundaries, a strided radius, the double-selection
error on the parallel route, ImageNet's 1.27 M rows x 1000 classes, and K6's margins past 2^31 elements.

Every case asserts the pick list element for element against the reference class loop (oracle.al_oracle.base_select at
small sizes, a device restatement of the same loop at large n, anchored to the oracle below), and asserts which route
ran from the launch counter: a parallel call is candidates + resolve, plus per fallback class the ordinary step (keys,
select_smallest, mark) and the resolve that resumes after it -- the fallback classes predicted by the twin
(tests/base_route_twin.py)."""
import numpy as np
import pytest
import torch

import base_route_twin as T
from oracle import al_oracle as O

pytestmark = pytest.mark.gpu

PER_CLASS_SMEM = T.LIST * 8 + 4            # one staged candidate list and its fail flag
EMPTY_S = (1 << 63) - 1                    # kBaseEmpty in the signed packing below
SMALL = 50000                              # up to this n the oracle's CPU loop is the reference


@pytest.fixture(scope="module")
def eng():
    from active_learning_b200.engine import Engine
    e = Engine()
    yield e
    e.set_option("base_impl", 0)


def optin():
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin


def bitset_bound():
    """Largest n whose taken-row bitset fits next to 8 staged lists and 1 KB of headroom."""
    return (optin() - 8 * PER_CLASS_SMEM - 1024) // 4 * 32


def chunk_of(n):
    return min(256, (optin() - 1024 - (n + 31) // 32 * 4) // PER_CLASS_SMEM)


def route_of(impl, n, c, budget):
    cnt_max = -(-budget // c)
    parallel = impl != 1 and cnt_max <= T.MAX_CNT and (c >= 16 or impl == 2) and n <= bitset_bound()
    return "parallel" if parallel else "sequential"


def to_device(K, seed=0):
    mm, radius, pred = T.split_keys(K, seed)
    return torch.from_numpy(mm).cuda(), torch.from_numpy(radius).cuda(), torch.from_numpy(pred).cuda()


def class_key(mm, radius, pred, k):
    return torch.where(pred == k, mm, radius[:, k])


def device_loop(mm, radius, pred, budget):
    """base_sampler.py:22-38 on the device with torch: per class the stable cnt smallest keys, taken rows at +inf."""
    n, c = radius.shape
    taken = torch.zeros(n, dtype=torch.bool, device=mm.device)
    out = []
    for k, cnt in enumerate(T.counts(budget, c)):
        if cnt == 0:
            continue
        key = class_key(mm, radius, pred, k).masked_fill(taken, float("inf"))
        idx = torch.sort(key, stable=True).indices[:int(cnt)]
        assert not taken[idx].any()
        taken[idx] = True
        out.append(idx)
    return torch.cat(out).cpu().numpy().astype(np.int64)


def reference(mm, radius, pred, budget):
    n, c = radius.shape
    if n <= SMALL:
        return O.base_select(mm.cpu(), radius.cpu(), pred.cpu().long(), budget, c)
    return device_loop(mm, radius, pred, budget)


def device_candidates(mm, radius, pred, budget, block=32):
    """T.candidates with torch on the device (the twin's lists and fail flags at any n): pairs packed as signed int64
    (ord - 2^31) * 2^32 + row, which orders like base_pack's unsigned words."""
    n, c = radius.shape
    cnt = T.counts(budget, c)
    m = max(-(-n // T.THREADS), T.KEEP + 1)
    rows = torch.arange(n, device=mm.device, dtype=torch.int64)
    lists = np.full((c, T.LIST), T.EMPTY, dtype=np.uint64)
    fail = np.zeros(c, dtype=bool)
    live = [k for k in range(c) if cnt[k]]
    for b0 in range(0, len(live), block):
        ks = live[b0:b0 + block]
        kt = torch.tensor(ks, device=mm.device)
        key = torch.where(pred[:, None] == kt[None, :], mm[:, None], radius[:, kt]).T.contiguous() + 0.0
        u = key.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
        o = torch.where(u >= (1 << 31), ~u & 0xFFFFFFFF, u | (1 << 31))
        w = torch.full((len(ks), m * T.THREADS), EMPTY_S, dtype=torch.int64, device=mm.device)
        w[:, :n] = (o - (1 << 31)) * (1 << 32) + rows
        s = w.view(len(ks), m, T.THREADS).sort(dim=1).values
        kept = s[:, :T.KEEP, :].reshape(len(ks), -1).sort(dim=1).values[:, :T.LIST]
        lens = torch.tensor([T.list_len(cnt[k]) for k in ks], device=mm.device)
        last = kept.gather(1, (lens - 1)[:, None])
        f = (s[:, T.KEEP, :] < last).any(dim=1)
        kept = torch.where(torch.arange(T.LIST, device=mm.device)[None, :] < lens[:, None], kept, EMPTY_S)
        lists[ks] = kept.cpu().numpy().view(np.uint64) ^ np.uint64(1 << 63)
        fail[ks] = f.cpu().numpy()
    return lists, fail


def twin_route(mm, radius, pred, budget):
    n, c = radius.shape
    lists, fail = device_candidates(mm, radius, pred, budget)
    picks, fallbacks, dup = T.resolve(lists, fail, lambda k: class_key(mm, radius, pred, k).cpu().numpy(), n, c, budget)
    return picks, fallbacks, fail, dup


_sel_cache = {}


def sel_launches(eng, n, budget, c):
    """select_smallest's launches for each per-class count of this call, measured with one call each."""
    out = {}
    for cnt in set(int(x) for x in T.counts(budget, c) if x):
        if (n, cnt) not in _sel_cache:
            x = torch.rand(n, device="cuda")
            l0 = eng.launches
            eng.select_smallest(x, cnt)
            _sel_cache[(n, cnt)] = eng.launches - l0
        out[cnt] = _sel_cache[(n, cnt)]
    return out


def run(eng, impl, mm, radius, pred, budget):
    eng.set_option("base_impl", impl)
    try:
        l0 = eng.launches
        got = eng.base_select(mm, radius, pred, budget).cpu().numpy().astype(np.int64)
        return got, eng.launches - l0
    finally:
        eng.set_option("base_impl", 0)


def check_routes(eng, mm, radius, pred, budget, impls=(0, 1, 2), ref=None, predict=True):
    """Every impl against the reference, and each call's launch delta against its route; returns the twin's
    (fallback classes, fail flags) (None, None) without a prediction."""
    n, c = radius.shape
    if ref is None:
        ref = reference(mm, radius, pred, budget)
    fallbacks = fail = None
    if predict:
        picks, fallbacks, fail, dup = twin_route(mm, radius, pred, budget)
        assert dup == 0 and picks.tolist() == ref.tolist()
    sel = sel_launches(eng, n, budget, c)
    for impl in impls:
        got, d = run(eng, impl, mm, radius, pred, budget)
        route = route_of(impl, n, c, budget)
        assert got.tolist() == ref.tolist(), (impl, route)
        if route == "parallel":
            want = T.launch_delta(fallbacks, c, budget, sel)
        else:
            want = T.sequential_delta(c, budget, sel)
            assert want >= 3 * int((T.counts(budget, c) > 0).sum())
        assert d == want, (impl, route, d, want, fallbacks)
    return fallbacks, fail


# ---------------------------------------------------------------------------------------------------------------
# the references themselves
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,c,budget,targets", [(3000, 20, 300, []), (4500, 1003, 3009, [0, 500, 1001, 1002]),
                                                (6000, 24, 23, [5]), (5000, 16, 512, [15])])
def test_device_restatements_match_the_oracle_and_the_twin(n, c, budget, targets):
    K = T.forced_fail(n, c, targets, n) if targets else T.random_keys(n, c, n, quantise=True)
    mm, radius, pred = to_device(K)
    want = O.base_select(mm.cpu(), radius.cpu(), pred.cpu().long(), budget, c)
    assert device_loop(mm, radius, pred, budget).tolist() == want.tolist()
    lists, fail = device_candidates(mm, radius, pred, budget)
    tl, tf = T.candidates(T.key_fn(K), c, budget)
    assert np.array_equal(lists, tl) and np.array_equal(fail, tf)
    assert np.flatnonzero(fail).tolist() == [k for k in targets if T.counts(budget, c)[k]]


# ---------------------------------------------------------------------------------------------------------------
# 1. forced fail flags
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,c,targets", [(6000, 20, [0, 7, 19]), (4500, 1003, [0, 500, 1001, 1002])])
def test_forced_fail_flags(eng, n, c, targets):
    """The 4 smallest keys of a class on one thread: the first class, the last class, and (C = 1003) the partial last
    8-class group of the candidates kernel."""
    budget = 3 * c
    mm, radius, pred = to_device(T.forced_fail(n, c, targets, 5))
    fallbacks, fail = check_routes(eng, mm, radius, pred, budget)
    assert np.flatnonzero(fail).tolist() == targets and fallbacks == targets


# ---------------------------------------------------------------------------------------------------------------
# 2. lists that run out
# ---------------------------------------------------------------------------------------------------------------
def test_exhausted_lists_fall_back_class_after_class(eng):
    c, budget = 100, 1000
    mm, radius, pred = to_device(T.exhausted(20000, c, 2))
    fallbacks, fail = check_routes(eng, mm, radius, pred, budget)
    assert not fail.any() and fallbacks == list(range(4, c))


def test_exhausted_only_at_the_last_class(eng):
    """The walk stops at c - 1: the ordinary step for the last class and no resolve after it."""
    c, cnt = 20, 10
    mm, radius, pred = to_device(T.exhausted_at(5000, c, cnt, 4))
    fallbacks, fail = check_routes(eng, mm, radius, pred, c * cnt)
    assert fallbacks == [c - 1] and not fail.any()


# ---------------------------------------------------------------------------------------------------------------
# 3. ties and +inf keys
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,c,budget,short", [(8000, 30, 300, 0), (20000, 64, 640, None), (4100, 17, 17 * 32, None)])
def test_ties_and_infinite_keys(eng, n, c, budget, short):
    K = T.ties(n, c, n + c, short_class=short, short_finite=4)
    mm, radius, pred = to_device(K)
    fallbacks, fail = check_routes(eng, mm, radius, pred, budget)
    if short is not None:
        assert fallbacks[0] == short


def test_random_quantised_pool(eng):
    mm, radius, pred = to_device(T.random_keys(30000, 200, 9, quantise=True))
    check_routes(eng, mm, radius, pred, 2000)


# ---------------------------------------------------------------------------------------------------------------
# 4. route boundaries
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c,route", [(15, "sequential"), (16, "parallel")])
def test_class_count_boundary_in_auto_mode(eng, c, route):
    assert route_of(0, 3000, c, 10 * c) == route
    mm, radius, pred = to_device(T.forced_fail(5000, c, [c - 2], c))
    fallbacks, _ = check_routes(eng, mm, radius, pred, 10 * c)
    assert fallbacks == [c - 2]


@pytest.mark.parametrize("c", [1, 8, 15])
def test_few_classes_on_the_parallel_route(eng, c):
    budget = 20 * c
    assert route_of(2, 5000, c, budget) == "parallel"
    mm, radius, pred = to_device(T.forced_fail(5000, c, [c - 1], c + 100))
    fallbacks, _ = check_routes(eng, mm, radius, pred, budget, impls=(2, 1))
    assert fallbacks == [c - 1]
    mm, radius, pred = to_device(T.random_keys(5000, c, c))
    check_routes(eng, mm, radius, pred, budget, impls=(2,))


@pytest.mark.parametrize("extra,route", [(0, "parallel"), (1, "sequential")])
def test_picks_per_class_boundary(eng, extra, route):
    c = 16
    budget = T.MAX_CNT * c + extra
    assert route_of(0, 6000, c, budget) == route == route_of(2, 6000, c, budget)
    mm, radius, pred = to_device(T.forced_fail(6000, c, [3], 6))
    check_routes(eng, mm, radius, pred, budget)


def test_budget_below_the_class_count(eng):
    c, budget = 40, 25
    mm, radius, pred = to_device(T.forced_fail(5000, c, [3, 30], 8))
    fallbacks, fail = check_routes(eng, mm, radius, pred, budget)
    assert fallbacks == [3]


@pytest.mark.parametrize("extra,route", [(0, "parallel"), (32, "sequential")])
def test_bitset_bound(eng, extra, route):
    """n at the largest pool whose bitset fits (8 staged lists at a time) and 32 rows past it.  At the bound a forced
    fallback sits in the second chunk, so the resumed resolve restages from a class past the first chunk."""
    n, c = bitset_bound() + extra, 24
    budget = 5 * c
    assert route_of(0, n, c, budget) == route == route_of(2, n, c, budget)
    if extra == 0:
        assert chunk_of(n) == 8
    K = T.forced_fail(n, c, [13], 17)
    mm, radius, pred = to_device(K)
    del K
    fallbacks, fail = check_routes(eng, mm, radius, pred, budget, predict=route == "parallel")
    if route == "parallel":
        assert fallbacks == [13]


def test_picks_in_the_last_partial_bitset_word(eng):
    """n % 32 = 4: the last 4 rows are the smallest keys of classes 0-5, class 0 takes them from its list, the others
    must find them taken in the last word -- also after class 2's fallback rebuilds the bitset from `taken`."""
    n, c = 4100, 20
    K = T.forced_fail(n, c, [2], 3)
    K[n - 4:, :6] = np.float32(1e-4) * np.arange(1, 5, dtype=np.float32)[:, None]
    mm, radius, pred = to_device(K)
    ref = reference(mm, radius, pred, 10 * c)
    assert set(ref[:10].tolist()) >= set(range(n - 4, n))
    fallbacks, _ = check_routes(eng, mm, radius, pred, 10 * c, ref=ref)
    assert fallbacks == [2]


# ---------------------------------------------------------------------------------------------------------------
# 5. strided radius
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("targets", [[], [5, 19]])
def test_strided_radius(eng, targets):
    n, c = 6000, 20
    mm, radius, pred = to_device(T.forced_fail(n, c, targets, 12) if targets else T.random_keys(n, c, 12))
    slab = torch.full((n, c + 4), float("nan"), device="cuda")
    slab[:, :c] = radius
    view = slab[:, :c]
    assert view.stride(0) == c + 4
    ref = reference(mm, radius, pred, 10 * c)
    fallbacks, _ = check_routes(eng, mm, view, pred, 10 * c, ref=ref)
    assert fallbacks == targets


# ---------------------------------------------------------------------------------------------------------------
# 6. double selection on the parallel route
# ---------------------------------------------------------------------------------------------------------------
def test_double_selection_raises_on_the_parallel_route(eng):
    from active_learning_b200._lib import AlqError
    c = 16
    ginv = eng.class_gap_inv(torch.ones(c, 8).cuda())
    mm, pred, radius = eng.mase_margins(torch.zeros(64, c).cuda(), ginv, want_per_class=True)
    assert torch.isinf(mm).all() and torch.isinf(radius).all()
    assert route_of(0, 64, c, 40) == "parallel"
    for impl in (0, 2):
        eng.set_option("base_impl", impl)
        try:
            with pytest.raises(AlqError, match="selected twice"):
                eng.base_select(mm, radius, pred, 40)
        finally:
            eng.set_option("base_impl", 0)
        with pytest.raises(AssertionError):
            O.base_select(mm.cpu(), radius.cpu(), pred.cpu().long(), 40, c)
        m2, r2, p2 = to_device(T.forced_fail(5000, c, [4], 21))       # the engine is usable right after
        check_routes(eng, m2, r2, p2, 40, impls=(impl,))


# ---------------------------------------------------------------------------------------------------------------
# 7. ImageNet scale, 8. K6 past 2^31 elements
# ---------------------------------------------------------------------------------------------------------------
def free_bytes():
    return torch.cuda.mem_get_info()[0]


def test_imagenet_scale(eng):
    """1 281 167 - 10 000 pool rows, 1000 classes, 10 picks each: several resolve chunks; once as built, once with
    three forced fallbacks in three different chunks."""
    n, c, budget = 1281167 - 10000, 1000, 10000
    need = 2 * n * c * 4 + (2 << 30)
    if free_bytes() < need:
        pytest.skip(f"needs {need} bytes of free device memory, {free_bytes()} are free")
    chunk = chunk_of(n)
    assert route_of(0, n, c, budget) == "parallel" and -(-c // chunk) >= 4
    g = torch.Generator(device="cuda").manual_seed(1281167)
    w = torch.randn(c, 64, device="cuda", generator=g) * 0.3
    logits = torch.randn(n, c, device="cuda", generator=g) * 2.0
    logits[: n // 2] = torch.round(logits[: n // 2] * 2) / 2           # quantised half: equal keys inside each class
    mm, pred, radius = eng.mase_margins(logits, eng.class_gap_inv(w), want_per_class=True)
    del logits
    assert int((mm[: n // 2] == 0).sum()) > 1000
    check_routes(eng, mm, radius, pred, budget)
    targets = [chunk // 2, chunk * 2 + 3, c - 5]
    assert len({k // chunk for k in targets}) == 3
    for k in targets:
        rows = torch.tensor([T.fail_row(k) + j * T.THREADS for j in range(4)], device="cuda")
        vals = -1.0 + 1e-3 * torch.arange(4, device="cuda", dtype=torch.float32)      # below every margin
        own = pred[rows] == k
        mm[rows[own]] = vals[own]
        radius[rows[~own], k] = vals[~own]
    fallbacks, fail = check_routes(eng, mm, radius, pred, budget)
    assert set(targets) <= set(np.flatnonzero(fail).tolist()) and set(targets) <= set(fallbacks)


def test_margins_past_2_31_elements_then_base_select(eng):
    """n x 1024 with n = 2 100 000: the radius matrix and the logits slab pass 2^31 floats at row 2 097 152.  The tail
    rows against the closed form, then base_select on the same tensors (the sequential route at this n)."""
    n, c = 2100000, 1024
    need = 2 * n * c * 4 + (1 << 30)
    if free_bytes() < need:
        pytest.skip(f"needs {need} bytes of free device memory, {free_bytes()} are free")
    first = (1 << 31) // c
    assert n * c > (1 << 31) and first < n
    g = torch.Generator(device="cuda").manual_seed(2100000)
    w = torch.randn(c, 48, device="cuda", generator=g) * 0.3
    logits = torch.randn(n, c, device="cuda", generator=g) * 2.0
    mm, pred, radius = eng.mase_margins(logits, eng.class_gap_inv(w), want_per_class=True)
    lo = first - 1000
    rmm, rpc, rpred = O.mase_margins_closed_form(logits[lo:].cpu(), w.cpu())
    del logits
    assert torch.equal(pred[lo:].cpu().long(), rpred)
    assert torch.equal(torch.isinf(radius[lo:].cpu()), torch.isinf(rpc))
    fin = torch.isfinite(rpc)
    torch.testing.assert_close(radius[lo:].cpu()[fin], rpc[fin], rtol=5e-6, atol=1e-30)
    torch.testing.assert_close(mm[lo:].cpu(), rmm, rtol=5e-6, atol=1e-30)
    budget = 2 * c
    assert route_of(0, n, c, budget) == "sequential"
    check_routes(eng, mm, radius, pred, budget, impls=(0,), predict=False)
