"""The sharded uncertainty tail (alq_uncertainty_tail_sharded) and its fallbacks at the edges the one-GPU fused tail is
held to, in a group of one rank on one GPU.  As in test_gpu_tail_one_rank.py, the peer-memory window is then this GPU's
own memory, and the fused launch runs select_epilogue_mgpu with the real stores, waits, fences and tags.

Every sharded result is checked against two references:
  * torch's stable sort of K1's own scores (NaN last, -0.0 == +0.0, ties by position): positions equal element for
    element, shifted by the shard's row offset; scores equal to score_softmax bit for bit;
  * the separate kernels, score_softmax + select_smallest.
Each call runs at row_lo = 0 and 2^30 + 7 and on both ranking routes (option tail_buckets 1 and 0).  After each call the
stream is synchronised and comm_check() must pass; the timing stamps must then say whether the fused launch ran, as
`helpers.fuses` predicts.

Not covered on one GPU: the cross-rank indexing (segments of ranks r > 0, the `level * W + rank` slots) and the overflow of
a rank's candidate region, which cannot happen at world size 1.  Those run only in test_gpu_multi.py, on two or more
GPUs."""
import contextlib

import numpy as np
import pytest
import torch

import row_reference as R
from helpers import fuses, make_strategy, one_rank_engine, tail_rows_per_tile, tied_tail_pools
from oracle import al_oracle as O
from test_gpu_row_kernels import MODE_NAMES, bits, check_within, special_scores
from test_oracle_golden import _same_selection
from test_row_reference import special_rows

pytestmark = pytest.mark.gpu

MODES = (0, 1, 2)
ROW_LO_BIG = (1 << 30) + 7      # global positions stay below 2^31 for every pool here
TOPB_WORDS = 16384              # the largest budget of alq_topb_exchange (AlqComm::kTopbWords)


@pytest.fixture(scope="module")
def eng(tmp_path_factory):
    with one_rank_engine(tmp_path_factory.mktemp("one_rank_group")) as e:
        yield e


@contextlib.contextmanager
def tail_buckets(eng, on):
    eng.set_option("tail_buckets", on)
    try:
        yield
    finally:
        eng.set_option("tail_buckets", 1)


def sm_count():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def stable_order(scores):
    return torch.sort(scores.cpu(), stable=True).indices.to(torch.int32)


def assert_path(eng, fused):
    """The last tail call took the fused launch (its %globaltimer stamps exist) or the separate kernels (no stamps)."""
    from active_learning_b200._lib import AlqError
    if fused:
        assert eng.uncertainty_tail_timing()[1] > 0
    else:
        with pytest.raises(AlqError, match="no fused launch"):
            eng.uncertainty_tail_timing()


def check_sharded(eng, logits, mode, budgets, fused=None):
    """Every b of `budgets` through the sharded tail on both routes and at both row offsets, against the stable sort and the
    separate kernels.  Returns K1's scores."""
    n, c = logits.shape
    fused = fuses(n, c) if fused is None else fused
    ref_s = eng.score_softmax(logits, mode)
    order = stable_order(ref_s)
    for b in budgets:
        assert torch.equal(eng.select_smallest(ref_s, b).cpu(), order[:b]), (n, c, mode, b)
        for buckets in (1, 0):
            with tail_buckets(eng, buckets):
                for row_lo in (0, ROW_LO_BIG):
                    s, p = eng.uncertainty_tail_sharded(logits, mode, b, row_lo, n, n)
                    torch.cuda.synchronize()
                    eng.comm_check()
                    assert_path(eng, fused)
                    assert torch.equal(bits(s), bits(ref_s)), (n, c, mode, b, buckets, row_lo)
                    assert torch.equal(p.cpu(), order[:b] + row_lo), (n, c, mode, b, buckets, row_lo)
    return ref_s


def nan_rows_pool(n, c, n_nan, seed):
    """The pool of test_fused_tail_with_nan_rows: randn * 3 logits, n_nan random rows with one NaN logit."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    logits = torch.randn(n, c, device="cuda", generator=g) * 3
    nan_rows = torch.randperm(n, generator=g, device="cuda")[:n_nan]
    logits[nan_rows, 17] = float("nan")
    return logits


@pytest.mark.parametrize("mode", MODES)
def test_sharded_tail_with_nan_rows(eng, mode):
    """NaN scores sort last in position order: b below, at and past the first NaN, and b = n (30 011 words, odd: the
    gathered list ends with a ~0 pad word)."""
    n, c, n_nan = 30011, 1000, 500
    s = check_sharded(eng, nan_rows_pool(n, c, n_nan, 5 + mode), mode,
                      (n - n_nan - 1, n - n_nan, n - n_nan + 1, n))
    assert int(torch.isnan(s).sum()) == n_nan


@pytest.mark.parametrize("mode", MODES)
def test_sharded_tail_with_nan_rows_inside_the_budget(eng, mode):
    """Most rows NaN (the first and the last row too), budgets that end inside the NaN group: the NaN words are
    candidates, alone in the last bin of both histogram levels (every finite score lies far below), and their count
    decides the threshold."""
    n, c = 20011, 64
    g = torch.Generator(device="cuda").manual_seed(41 + mode)
    logits = torch.randn(n, c, device="cuda", generator=g) * 3
    nan = torch.rand(n, device="cuda", generator=g) < 0.6
    nan[0] = nan[-1] = True
    logits[nan, 5] = float("nan")
    n_nan = int(nan.sum())
    n_fin = n - n_nan
    s = check_sharded(eng, logits, mode, (n_fin, n_fin + 1, n_fin + n_nan // 2, n - 1, n))
    assert torch.equal(stable_order(s)[n_fin:], torch.nonzero(nan.cpu()).flatten().to(torch.int32))


def tie_straddling_budgets(sorted_scores):
    """1 and n, around the first NaN, and a budget that cuts each of the three largest tie groups of finite scores
    (-0.0 and +0.0 tie)."""
    v = sorted_scores.numpy()
    n = len(v)
    first_nan = int(np.flatnonzero(np.isnan(v))[0]) if np.isnan(v).any() else n
    starts = np.flatnonzero(np.r_[True, v[1:first_nan] != v[:first_nan - 1]])
    sizes = np.diff(np.r_[starts, first_nan])
    cuts = {int(starts[i] + sizes[i] // 2) for i in np.argsort(-sizes, kind="stable")[:3] if sizes[i] > 1}
    return sorted(b for b in {1, n, first_nan - 1, first_nan, first_nan + 1, *cuts} if 1 <= b <= n)


@pytest.mark.parametrize("c", [12, 1000])
def test_sharded_tail_with_special_rows(eng, c):
    """test_row_reference.special_rows at the head of a fused-size pool and copied to every 50th row after it: masked
    classes, one finite logit, all -inf, NaN, +inf, +-3e38, gaps below -87, ties at the maximum.  One-hot entropies and
    margin ties give tie groups of zeros (+-0.0 in torch's stable sort: equal).  Scores of the special rows and of a
    sample are within the fp64 bound."""
    n = 30011
    rng = np.random.default_rng(c)
    z = (rng.standard_normal((n, c)) * 3).astype(np.float32)
    sp = special_rows(c, rng)
    z[:len(sp)] = sp
    copies = z[len(sp)::50]
    copies[:] = sp[np.arange(len(copies)) % len(sp)]
    logits = torch.from_numpy(z).cuda()
    rows = np.unique(np.r_[np.arange(len(sp)), rng.choice(n, 200, replace=False)])
    for mode in MODES:
        ref_s = eng.score_softmax(logits, mode)
        budgets = tie_straddling_budgets(torch.sort(ref_s.cpu(), stable=True).values)
        s = check_sharded(eng, logits, mode, budgets, fused=True)
        check_within(MODE_NAMES[mode], s.cpu().numpy()[rows], R.softmax_scores64(z[rows], mode),
                     R.score_bound(z[rows], mode, "vec"))


def register_width(c):
    """NV of the rows_pipe_kernel instantiation launch_rows_pipe_nv picks: ceil(c / 128) rounded up to 1, 2, 4, 8, 16."""
    need = -(-c // 128)
    return next(v for v in (1, 2, 4, 8, 16) if v >= need)


@pytest.mark.parametrize("c,nv", [(4, 1), (64, 1), (128, 1), (132, 2), (260, 4), (516, 8), (1024, 8), (2048, 16)])
def test_sharded_tail_at_every_register_width(eng, c, nv):
    """The sharded epilogue behind every NV instantiation (c = 2048: the spilling NV = 16 one), b from 1 to n; scores of
    a sample within the fp64 bound."""
    n = 30011
    assert register_width(c) == nv and fuses(n, c)
    g = torch.Generator(device="cuda").manual_seed(c)
    logits = torch.randn(n, c, device="cuda", generator=g) * 3
    sub = np.random.default_rng(c).choice(n, 200, replace=False)
    zs = logits[torch.from_numpy(sub).cuda()].cpu().numpy()
    for mode in MODES:
        s = check_sharded(eng, logits, mode, (1, 777, n // 3, n), fused=True)
        check_within(MODE_NAMES[mode], s.cpu().numpy()[sub], R.softmax_scores64(zs, mode), R.score_bound(zs, mode, "vec"))


@pytest.mark.parametrize("c", [12, 1000])
def test_sharded_fusing_boundary(eng, c):
    """The sharded launch fuses when the one-GPU rule holds (4096 <= n, 5 n <= sm * 2048 * 4) and the shard has at least
    one row tile per SM.  On each side of each boundary the result is the same, and the timing stamps say which path ran
    (the other side is K1 + K1b + alq_topb_exchange).  A budget above the exchange's 16 384 words is served by the fused
    launch; where the launch does not fuse it is declined before anything runs."""
    from active_learning_b200._lib import AlqError
    sm = sm_count()
    rows = tail_rows_per_tile(c)
    n_tile = (sm - 1) * rows + 1                    # the smallest shard with one row tile per SM
    n_max = sm * 2048 * 4 // 5
    edges = [(n_max + 1, n_max), (n_tile - 1, n_tile) if n_tile > 4096 else (4095, 4096)]    # (split, fused)
    for off, on in edges:
        assert not fuses(off, c) and fuses(on, c), (c, off, on)
    g = torch.Generator(device="cuda").manual_seed(c + 3)
    big = torch.randn(n_max + 1, c, device="cuda", generator=g) * 3
    for n in sorted({n_tile - 1, n_tile, *(x for e in edges for x in e)}):
        for mode in MODES:
            check_sharded(eng, big[:n], mode, (min(777, n), min(n // 2, TOPB_WORDS)))
    check_sharded(eng, big[:n_max], 1, (TOPB_WORDS + 1, n_max // 2))
    launches = eng.launches
    with pytest.raises(AlqError, match="does not fuse"):
        eng.uncertainty_tail_sharded(big, 1, TOPB_WORDS + 1, 0, n_max + 1, n_max + 1)
    assert eng.launches == launches


def test_sharded_calls_in_a_row(eng):
    """Sharded calls back to back without a synchronise.  The window regions are double-buffered by call parity, so each
    call reuses the region of the call two epochs before it: a small budget (few candidates) follows large ones whose
    thousands of candidate words (a huge tie group at the threshold) are still in that region, with modes, row offsets,
    a direct alq_topb_exchange and a sharded call that does not fuse in between.  Every result equals the separate
    kernels after the last call."""
    big, b_big = list(tied_tail_pools())[1]            # 150 000 x 4 dyadic logits, b = 12 000
    g = torch.Generator(device="cuda").manual_seed(8)
    small = torch.randn(30011, 64, device="cuda", generator=g) * 3
    split = torch.randn((sm_count() - 1) * tail_rows_per_tile(12) - 5, 12, device="cuda", generator=g) * 3
    assert fuses(*big.shape) and fuses(*small.shape) and not fuses(*split.shape)
    xs = torch.from_numpy(special_scores(9000, 3)).cuda()
    xpos = eng.select_smallest(xs, 3000)
    calls = [(big, 0, b_big), (big, 1, b_big), (small, 2, 50), (small, 0, 50), ("exchange", None, 3000), (big, 2, b_big),
             (split, 1, 700), (small, 1, 50), (small, 2, 50), (big, 0, b_big)]
    for buckets in (1, 0):
        with tail_buckets(eng, buckets):
            outs = []
            for k, (x, mode, b) in enumerate(calls):
                row_lo = ROW_LO_BIG if k % 2 else 0
                if isinstance(x, str):
                    outs.append(eng.topb_exchange(xs, xpos, row_lo, b))
                else:
                    outs.append(eng.uncertainty_tail_sharded(x, mode, b, row_lo, len(x), len(x))[1])
            torch.cuda.synchronize()
            eng.comm_check()
            assert_path(eng, True)
            for k, ((x, mode, b), got) in enumerate(zip(calls, outs)):
                row_lo = ROW_LO_BIG if k % 2 else 0
                ref = xpos if isinstance(x, str) else eng.select_smallest(eng.score_softmax(x, mode), b)
                assert torch.equal(got, ref + row_lo), (buckets, k)


def test_topb_exchange_with_special_scores(eng):
    """alq_topb_exchange at world size 1 on scores with NaN, -NaN, +-inf, +-0 and ties: the local winners come back as
    global positions in stable-sort order, also when the shard has fewer rows than b (a list padded with ~0 words) and at
    b = 16 384, the largest budget ShardGroup.merge_smallest sends through it."""
    from active_learning_b200._lib import AlqError
    s = torch.from_numpy(special_scores(40000, 9)).cuda()
    for n, b in ((40000, 1), (40000, 777), (40000, TOPB_WORDS), (1, 3), (300, 301), (5001, TOPB_WORDS)):
        loc = s[:n].contiguous()
        k = min(n, b)
        pos = eng.select_smallest(loc, k)
        assert torch.equal(pos.cpu(), stable_order(loc)[:k]), (n, b)
        for row_lo in (0, ROW_LO_BIG):
            out = eng.topb_exchange(loc, pos, row_lo, b)
            torch.cuda.synchronize()
            eng.comm_check()
            assert torch.equal(out[:k].cpu(), pos.cpu() + row_lo), (n, b, row_lo)
    with pytest.raises(AlqError):
        eng.topb_exchange(s, eng.select_smallest(s, TOPB_WORDS + 1), 0, TOPB_WORDS + 1)


@pytest.mark.parametrize("bounds", [(0, 1234, 40000, 100003), (0, 7, 20000, 20500, 70000, 100003)])
def test_topb_pack_merge_with_special_scores_and_padded_shards(eng, bounds):
    """The primitives of ShardGroup.merge_smallest's collective path, without the collective: one score vector with NaN,
    -NaN, +-inf, +-0 and massive ties cut into 3 and 5 uneven shards, some shorter than b (packed with ~0 padding), packed
    to b_pad = b and b + 37 words, merged with list_len 0 (sort) and b_pad (sorted lists).  Budgets up to n, past the
    16 384 words the window exchange takes.  The result is torch's stable sort of the whole vector."""
    n = bounds[-1]
    s = torch.from_numpy(special_scores(n, 17)).cuda()
    order = stable_order(s)
    for b in (1, 5000, TOPB_WORDS + 1, 40000, n):
        for base in (0, ROW_LO_BIG):
            winners = []
            for lo, hi in zip(bounds[:-1], bounds[1:]):
                loc = s[lo:hi].contiguous()
                winners.append((loc, eng.select_smallest(loc, min(b, hi - lo)), base + lo))
            for b_pad in (b, b + 37):
                keys = torch.cat([eng.topb_pack(loc, pos, lo, b_pad) for loc, pos, lo in winners])
                for list_len in (0, b_pad):
                    got = eng.topb_merge(keys, b, list_len=list_len)
                    assert torch.equal(got.cpu(), order[:b] + base), (b, base, b_pad, list_len)


def sharded_query(eng, s, budget, seed):
    """UncertaintyQuery._query_sharded with a one-rank ShardGroup (query() takes it only for world_size > 1), next to the
    unsharded _tail path on the same pool.  Returns (pool indices, sharded positions, unsharded positions, fused)."""
    from active_learning_b200._lib import AlqError
    from active_learning_b200.sharding import ShardGroup
    s._shard_group = ShardGroup()
    np.random.seed(seed)
    idxs = s.available_query_idxs(boolean=False, shuffle=s.SHUFFLE_POOL)
    budget = int(min(len(idxs), budget))
    pos = s._query_sharded(idxs, budget, s._shard_group)
    try:
        eng.uncertainty_tail_timing()
        fused = True
    except AlqError:
        fused = False
    logits, _ = s._forward_pool(idxs, s.net, want_features=False)
    ref = s._tail(eng, logits, budget)[1].cpu().numpy()
    assert pos.dtype == np.int64 and np.array_equal(pos, ref), (type(s).__name__, budget)
    return idxs, pos, fused, logits.shape


def test_samplers_sharded_branch_on_the_goldens(eng, gold):
    """Margin, Confidence and Entropy through _query_sharded on the golden pools (700 rows: the launch does not fuse and
    alq_topb_exchange serves the query): the positions of the unsharded path and the reference's recorded picks (on the
    dyadic pools the reference's unstable sort orders ties its own way: same score sequence, stable tie-break here)."""
    n, ev, lab = int(gold["e2e_n"]), gold["e2e_eval_idxs"], gold["e2e_labeled"]
    cases = [("MarginSampler", "margin_f32_c10"), ("MarginSampler", "margin_f32_c1000"),
             ("MarginSampler", "margin_dyadic_c10"), ("ConfidenceSampler", "confidence_f32"),
             ("ConfidenceSampler", "confidence_dyadic"), ("EntropySampler", "margin_f32_c1000")]
    for name, tag in cases:
        logits = torch.from_numpy(gold[f"{tag}_logits"])
        s = make_strategy(name, logits, torch.zeros(n, 4), ev, lab, 128, engine=eng)
        idxs, pos, fused, _ = sharded_query(eng, s, 60.0, 7)
        assert not fused
        if name != "EntropySampler":            # the reference has no entropy sampler: no recorded picks
            _same_selection(idxs[pos].tolist(), gold[f"{tag}_picks"].tolist(), idxs,
                            O.softmax_scores(logits[idxs], s.MODE), exact_order="dyadic" not in tag)


@pytest.mark.parametrize("pool", ["nan", "split"])
def test_samplers_sharded_branch_on_large_pools(eng, pool):
    """The same on a fused-size pool with NaN rows (the budget reaches into them) and on a pool with fewer row tiles than
    SMs, which alq_uncertainty_tail_sharded serves through its own alq_topb_exchange."""
    g = torch.Generator().manual_seed(12)
    if pool == "nan":
        n, c, budget = 20000, 64, 19705
        logits = torch.randn(n, c, generator=g) * 3
        logits[torch.randperm(n, generator=g)[:300], 9] = float("nan")
    else:
        n, c, budget = (sm_count() - 1) * tail_rows_per_tile(12) - 5, 12, 700
        logits = torch.randn(n, c, generator=g) * 3
    for name in ("MarginSampler", "ConfidenceSampler", "EntropySampler"):
        s = make_strategy(name, logits, torch.zeros(n, 4), [], [], 4096, engine=eng)
        _, _, fused, shape = sharded_query(eng, s, budget, 3)
        assert fused == (pool == "nan") == fuses(*shape), name
