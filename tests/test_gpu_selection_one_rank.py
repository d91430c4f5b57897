"""The global CoreSet / BADGE selection loop's group path (alq_greedy_desc.shard_off_host) in a group of one rank.

One GPU: a gloo group of world size 1 (helpers.one_rank_engine).  The peer-memory window is then this GPU's own memory,
but a call with shard_off = [0, n] (and, for the D^2 draw, shard_pos = [0, full_n]) runs the group path: the words in
the window instead of scratch, the window's size check, shard_pos turned into leaf bounds, the ready handshake
(alq_comm_ready + the kernel's ready wait) and the epoch-tagged words in the window region that K11 and K12 also use.  It
must return the picks of the same call without shard_off on the same engine, bit for bit, and CoresetQuery's
_query_global_sharded must return the goldens that test_gpu_multi.py checks on two GPUs.

Not covered here, only with two or more GPUs (test_gpu_multi.py): other ranks' segments in the segment table, leaf
masses summed across ranks, and a D^2 crossing inside another rank's rows.  Two ranks are not emulated on one GPU: two
persistent launches are not guaranteed to run at the same time, so one would sit in its bounded wait."""
import numpy as np
import pytest
import torch

from helpers import make_strategy, one_rank_engine
from test_balancing_loop import _state_equal
from test_gpu_balancing_loop import make_pool
from test_gpu_balancing_table import option
from test_gpu_greedy import _assert_prefix_parity

pytestmark = pytest.mark.gpu

L2_DEFAULT_MB = 24          # alq_ctx's l2_resident_mb default
KINDS = {"dense": 0, "c10": 10, "c1000": 1000}     # factored BADGE rows: c classes, padded to a multiple of 4


@pytest.fixture(scope="module")
def eng(tmp_path_factory):
    with one_rank_engine(tmp_path_factory.mktemp("selection_one_rank")) as e:
        yield e


@pytest.fixture(scope="module")
def plain():
    from active_learning_b200.engine import Engine
    e = Engine()
    yield e
    e.close()


@pytest.fixture(scope="module")
def group(eng):
    from active_learning_b200.sharding import ShardGroup
    return ShardGroup()


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


class Problem:
    """One selection problem on the device: n candidate rows of width d (plus factors of c classes), the running
    min-distance of a labeled start or of a cold start (first_pick), and the D^2 draw's positions in the full array."""

    def __init__(self, eng, n, d, c, seed, cold):
        rng = np.random.default_rng(seed)
        self.n = n
        self.x = torch.from_numpy(rng.standard_normal((n, d), dtype=np.float32)).cuda()
        self.xn = eng.row_norm2(self.x)
        self.a = self.an = None
        if c:
            a = np.zeros((n, (c + 3) & ~3), dtype=np.float32)
            a[:, :c] = rng.standard_normal((n, c), dtype=np.float32) * 0.3
            self.a = torch.from_numpy(a).cuda()
            self.an = eng.row_norm2(self.a)
        n_lab = 0 if cold else 7
        self.full_n = n + n_lab
        self.vpos = torch.from_numpy(np.sort(rng.choice(self.full_n, n, replace=False)).astype(np.int32)).cuda()
        self.first = int(rng.integers(n)) if cold else None
        self.mind = torch.full((n,), float("inf"), device="cuda")
        if n_lab:
            y = torch.from_numpy(rng.standard_normal((n_lab, d), dtype=np.float32)).cuda()
            ya = yan = None
            if c:
                ya = torch.from_numpy(np.pad(rng.standard_normal((n_lab, c), dtype=np.float32) * 0.3,
                                             ((0, 0), (0, self.a.shape[1] - c)))).cuda()
                yan = eng.row_norm2(ya)
            eng.min_dist(self.x, self.xn, y, eng.row_norm2(y), self.a, self.an, ya, yan, out=self.mind)
        self.rng = rng

    def call(self, eng, budget, sample, sharded, us=None, **kw):
        """-> (picks, mind afterwards) of one greedy_select on a copy of the start's min-distances."""
        mind = self.mind.clone()
        args = dict(a=self.a, an=self.an, first_pick=[self.first] if self.first is not None else None)
        if sample:
            args.update(uniforms=us, vpos=self.vpos, full_n=[self.full_n])
        if sharded:
            args.update(shard_off=[0, self.n], shard_pos=[0, self.full_n] if sample else None)
        args.update(kw)
        picks = eng.greedy_select(self.x, self.xn, mind, [0, self.n], [budget], **args)
        return picks.tolist(), mind

    def twins(self, eng, budget, sample):
        """The sharded call and the same call without shard_off must agree bit for bit (picks and min-distances)."""
        us = self.rng.random(budget) if sample else None
        one, m1 = self.call(eng, budget, sample, False, us)
        grp, m2 = self.call(eng, budget, sample, True, us)
        assert grp == one, (self.n, budget, sample)
        assert torch.equal(m1.view(torch.int32), m2.view(torch.int32))
        assert len(set(grp)) == budget
        return grp


def _shapes(sms):
    """(n, d, budgets): empty and one-row CTA segments, a few thousand rows, and a run of steps well past 4 096 (the
    12-bit round of the arg-max key tags wraps)."""
    out = [(n, 36, sorted({1, min(n, 3), n})) for n in (1, 2, sms - 1, sms, sms + 1)]
    out += [(3000, 4, [1, 300]), (3000, 36, [1, 3000]), (2000, 2048, [1, 300]), (6000, 4, [5000])]
    return out


@pytest.mark.parametrize("l2_mb", [0, L2_DEFAULT_MB])
@pytest.mark.parametrize("cold", [False, True], ids=["labeled", "cold"])
@pytest.mark.parametrize("mode", ["argmax", "d2_fast", "d2_exact"])
@pytest.mark.parametrize("kind", list(KINDS))
def test_group_path_equals_single_gpu_loop(eng, sms, kind, mode, cold, l2_mb):
    sample = mode != "argmax"
    try:
        eng.set_option("l2_resident_mb", l2_mb)
        eng.set_option("d2_fast_path", int(mode != "d2_exact"))
        for i, (n, d, budgets) in enumerate(_shapes(sms)):
            p = Problem(eng, n, d, KINDS[kind], 1000 * i + n + d, cold)
            for b in budgets:
                p.twins(eng, b, sample)
    finally:
        eng.set_option("l2_resident_mb", L2_DEFAULT_MB)
        eng.set_option("d2_fast_path", 1)


# ------------------------------------------------------------------------------------------- goldens through the group
def _golden_run(eng, feat, ind, b, sharded, randomize=False, us=None, first=None):
    """Reference-shaped call (test_gpu_greedy.py's): dense rows, labeled indicator -> picks as rows of feat."""
    cand, lab = np.flatnonzero(~ind), np.flatnonzero(ind)
    X = feat[cand].cuda()
    xn = eng.row_norm2(X)
    mind = torch.full((len(cand),), float("inf"), device="cuda")
    if len(lab):
        Y = feat[lab].cuda()
        eng.min_dist(X, xn, Y, eng.row_norm2(Y), out=mind)
    kw = {}
    if sharded:
        kw = dict(shard_off=[0, len(cand)], shard_pos=[0, len(ind)] if randomize else None)
    picks = eng.greedy_select(X, xn, mind, [0, len(cand)], [b], uniforms=us if randomize else None,
                              vpos=torch.as_tensor(cand.astype(np.int32)).cuda() if randomize else None,
                              full_n=[len(ind)] if randomize else None,
                              first_pick=[first] if first is not None else None, **kw)
    return cand[picks].tolist()


def _golden_twins(eng, feat, ind, b, **kw):
    outs = []
    for fast in ((1, 0) if kw.get("randomize") else (1,)):
        eng.set_option("d2_fast_path", fast)
        try:
            one = _golden_run(eng, feat, ind, b, False, **kw)
            grp = _golden_run(eng, feat, ind, b, True, **kw)
        finally:
            eng.set_option("d2_fast_path", 1)
        assert grp == one
        outs.append(grp)
    assert all(o == outs[0] for o in outs)
    return outs[0]


@pytest.mark.parametrize("tag", ["int", "f32"])
def test_group_path_replays_the_greedy_and_kmeanspp_goldens(eng, gold, tag):
    feat, ind = torch.from_numpy(gold[f"cs_{tag}_feat"]), gold["cs_indicator"]
    got = _golden_twins(eng, feat, ind, 40)
    if tag == "int":
        assert got == gold["cs_int_greedy"].tolist()
    else:
        _assert_prefix_parity(got, gold["cs_f32_greedy"].tolist(), feat, ind, False)
    np.random.seed(11)
    us = np.random.random_sample(40)
    assert _golden_twins(eng, feat, ind, 40, randomize=True, us=us) == gold[f"cs_{tag}_d2sample"].tolist()
    # cold starts: the minimax centre, and np.random.choice's centre for k-means++
    none = np.zeros(len(feat), dtype=bool)
    X = feat.cuda()
    xn = eng.row_norm2(X)
    q0 = eng.argmin(eng.min_dist(X, xn, X, xn, reduce_max=True))
    assert _golden_twins(eng, feat, none, 6, first=q0) == gold[f"cs_{tag}_greedy_cold"].tolist()
    np.random.seed(12)
    q0 = int(np.random.choice(len(feat)))
    us = np.zeros(6)
    us[1:] = np.random.random_sample(5)
    assert _golden_twins(eng, feat, none, 6, randomize=True, us=us, first=q0) == gold[f"cs_{tag}_d2sample_cold"].tolist()


def test_group_path_replays_the_nan_retry_golden(eng, gold):
    """Every candidate duplicates a labeled row: sum(prob) == 0 -> NaN -> the `+= 1e-5` retry, through the window."""
    feat, ind = torch.from_numpy(gold["cs_dup_feat"]), gold["cs_dup_indicator"]
    np.random.seed(13)
    us = np.random.random_sample(5)
    assert _golden_twins(eng, feat, ind, 5, randomize=True, us=us) == gold["cs_dup_d2sample"].tolist()


# ------------------------------------------------------------------------------------------- the sharded query
E2E_RUNS = [("CoresetSampler", "all", {}),
            ("CoresetSampler", "sub", dict(subset_labeled=60, subset_unlabeled=300)),
            ("BADGESampler", "sub", dict(subset_labeled=60, subset_unlabeled=300))]


def _sharded_query(s, group, budget):
    """CoresetQuery.query up to its branch, then the sharded branch itself (query() takes it only for two or more ranks)."""
    union = np.asarray(s.get_idxs_for_coreset(), dtype=np.int64)
    return s._query_global_sharded(union, budget, group)


@pytest.mark.parametrize("etag", ["int", "f32"])
def test_sharded_query_returns_the_two_gpu_goldens(eng, plain, group, gold, etag):
    lg, emb = torch.from_numpy(gold["e2e_logits"]), torch.from_numpy(gold[f"e2e_emb_{etag}"])
    ev, lab = gold["e2e_eval_idxs"], gold["e2e_labeled"]
    for name, sub, kw in E2E_RUNS:
        s = make_strategy(name, lg, emb, ev, lab, 64, engine=eng, **kw)
        s._shard_group = group
        np.random.seed(21)
        idx, cost = _sharded_query(s, group, 50.0)
        state = np.random.get_state()
        assert [int(i) for i in idx] == gold[f"e2e_{name}_{sub}_{etag}"].tolist(), (name, sub)
        assert cost == len(idx)
        t = make_strategy(name, lg, emb, ev, lab, 64, engine=plain, **kw)
        np.random.seed(21)
        ref, _ = t.query(50.0)
        assert [int(i) for i in ref] == [int(i) for i in idx]
        assert _state_equal(np.random.get_state(), state), (name, sub)


@pytest.mark.parametrize("name", ["CoresetSampler", "BADGESampler"])
def test_sharded_query_cold_start_equals_single_gpu(eng, plain, group, gold, name):
    """Nothing labeled: the minimax centre through far_all (CoreSet) or np.random.choice's centre (BADGE)."""
    lg, emb, ev = torch.from_numpy(gold["e2e_logits"]), torch.from_numpy(gold["e2e_emb_int"]), gold["e2e_eval_idxs"]
    s = make_strategy(name, lg, emb, ev, [], 64, engine=eng)
    s._shard_group = group
    np.random.seed(5)
    idx, cost = _sharded_query(s, group, 12.0)
    state = np.random.get_state()
    t = make_strategy(name, lg, emb, ev, [], 64, engine=plain)
    np.random.seed(5)
    ref, _ = t.query(12.0)
    assert [int(i) for i in idx] == [int(i) for i in ref] and cost == 12
    assert _state_equal(np.random.get_state(), state)


# ------------------------------------------------------------------------------------------- one window, many kernels
def test_one_window_many_kernels_many_epochs(eng):
    """260 sharded calls that alternate the selection loop (dense arg-max, factored D^2), K11, K12 and the fused sharded
    tail on one window: every call bumps the group's epoch, so the key tags' 3 epoch bits (period 8) and tag_base's 7
    bits (period 128) both wrap.  Each result must equal its unsharded twin."""
    from helpers import fuses
    dense = Problem(eng, 3000, 16, 0, 1, False)
    fact = Problem(eng, 2500, 8, 12, 2, False)
    us = np.random.default_rng(3).random(60)
    want_dense = dense.call(eng, 40, False, False)[0]
    want_fact = fact.call(eng, 60, True, False, us)[0]
    emb, ys, avail, lab = make_pool(3000, 32, 6, 4, [30, 15, 8, 4, 2, 1])
    x = torch.from_numpy(emb).cuda()
    bargs = (x, eng.row_norm2(x), torch.from_numpy(ys.astype(np.int32)).cuda(), torch.from_numpy(avail.astype(np.uint8)).cuda(),
             torch.from_numpy(lab.astype(np.uint8)).cuda(), 6, 40)

    def balancing(opt, sharded):
        np.random.seed(8)
        with option(eng, opt):
            fn = eng.balancing_select if opt == 2 else eng.balancing_table_select
            res = fn(*bargs, **({"shard_off": [0, 3000]} if sharded else {}))
        return res[0].tolist(), res[1], np.random.get_state()

    want_bal = {opt: balancing(opt, False) for opt in (2, 3)}
    logits = torch.randn(8192, 12, device="cuda", generator=torch.Generator(device="cuda").manual_seed(9))
    assert fuses(8192, 12)
    want_tail = eng.select_smallest(eng.score_softmax(logits, 0), 100)
    calls = 0
    while calls < 260:
        assert dense.call(eng, 40, False, True)[0] == want_dense, calls
        assert fact.call(eng, 60, True, True, us)[0] == want_fact, calls
        for opt in (2, 3):
            got = balancing(opt, True)
            assert got[0] == want_bal[opt][0] and got[1] == want_bal[opt][1] and _state_equal(got[2], want_bal[opt][2])
        _, pos = eng.uncertainty_tail_sharded(logits, 0, 100, 0, 8192, 8192)
        assert torch.equal(pos, want_tail), calls
        calls += 5
    torch.cuda.synchronize()
    eng.comm_check()


# ------------------------------------------------------------------------------------------- the handshake is issued
@pytest.mark.parametrize("sample", [False, True], ids=["argmax", "d2"])
@pytest.mark.parametrize("c", [0, 10])
def test_group_path_issues_the_ready_handshake(eng, sample, c):
    """The persistent loop's launches plus exactly one: comm_ready_kernel, the ready word stored into the window."""
    p = Problem(eng, 5000, 64, c, 4, False)
    us = np.random.default_rng(5).random(30)
    counts = []
    for sharded in (False, True):
        before = eng.launches
        p.call(eng, 30, sample, sharded, us if sample else None)
        counts.append(eng.launches - before)
    assert counts[1] == counts[0] + 1, counts


# ------------------------------------------------------------------------------------------- host-side refusals
def _refused(eng, match, fn):
    """fn() raises AlqError matching `match` before anything is launched."""
    from active_learning_b200._lib import AlqError
    before = eng.launches
    with pytest.raises(AlqError, match=match):
        fn()
    assert eng.launches == before


def test_group_path_refusals_leave_the_context_usable(eng):
    from active_learning_b200.sharding import pairwise_leaf_bounds
    p = Problem(eng, 2000, 16, 0, 6, False)
    us = np.random.default_rng(7).random(20)
    want_d2 = p.call(eng, 20, True, False, us)[0]
    want_max = p.call(eng, 20, False, False)[0]
    lb = eng.leaf_bounds(p.full_n)
    assert lb.tolist() == pairwise_leaf_bounds(p.full_n).tolist() and len(lb) > 3
    off_leaf = int(lb[1]) + 1
    assert off_leaf not in set(lb.tolist())
    bad_calls = [
        ("shard_pos", dict(shard_pos=None)),                                   # D^2 without shard_pos
        ("shard_pos", dict(shard_pos=[0, p.full_n - 1])),                      # the end off a leaf boundary
        ("shard_pos", dict(shard_pos=[off_leaf, p.full_n])),                   # the start off a leaf boundary
        ("shard_pos", dict(shard_pos=[int(lb[1]), p.full_n])),                 # a leaf boundary, but not [0, full_n]
    ]
    for match, kw in bad_calls:
        _refused(eng, match, lambda: p.call(eng, 20, True, True, us, **kw))
        assert p.call(eng, 20, True, True, us)[0] == want_d2
    # two partitions
    half = p.n // 2
    _refused(eng, "one global partition",
             lambda: eng.greedy_select(p.x, p.xn, p.mind.clone(), [0, half, p.n], [5, 5], shard_off=[0, p.n]))
    assert p.call(eng, 20, False, True)[0] == want_max
    # the per-step variants
    for variant in (1, 2):
        _refused(eng, "the multi-GPU loop has no other variant", lambda: p.call(eng, 20, False, True, variant=variant))
        _refused(eng, "the multi-GPU loop has no other variant", lambda: p.call(eng, 20, True, True, us, variant=variant))
        assert p.call(eng, 20, False, True)[0] == want_max
    try:
        eng.set_option("greedy_variant", 2)
        _refused(eng, "the multi-GPU loop has no other variant", lambda: p.call(eng, 20, False, True))
    finally:
        eng.set_option("greedy_variant", 0)
    assert p.call(eng, 20, False, True)[0] == want_max


def test_group_path_refuses_a_segment_past_the_key_word(eng, sms):
    """Arg-max key words carry a 16-bit row offset: 65 535 rows per CTA is the most a shard of one rank can stream.  One
    row more is refused by name (one GPU falls back to the per-step kernels; the group path has no fallback)."""
    n = 65535 * sms
    g = torch.Generator(device="cuda").manual_seed(11)
    x = torch.rand(n + 1, 4, device="cuda", generator=g)
    xn = eng.row_norm2(x)
    mind0 = torch.rand(n + 1, device="cuda", generator=g) * 4
    one = eng.greedy_select(x[:n], xn[:n], mind0[:n].clone(), [0, n], [3])
    grp = eng.greedy_select(x[:n], xn[:n], mind0[:n].clone(), [0, n], [3], shard_off=[0, n])
    assert grp.tolist() == one.tolist()
    _refused(eng, "the multi-GPU loop has no other variant",
             lambda: eng.greedy_select(x, xn, mind0.clone(), [0, n + 1], [3], shard_off=[0, n + 1]))
    assert eng.greedy_select(x[:n], xn[:n], mind0[:n].clone(), [0, n], [3], shard_off=[0, n]).tolist() == one.tolist()


def test_group_path_refuses_a_window_too_small(eng):
    """A second context in the same group with a 64 KB window: the group path's words do not fit (ALQ_ERR_NOMEM) before
    anything runs, and the same context's call without shard_off still returns the single-GPU picks."""
    from active_learning_b200.engine import Engine
    small = Engine().comm_init(window_bytes=1 << 16)
    try:
        p = Problem(small, 3000, 16, 0, 8, False)
        us = np.random.default_rng(9).random(25)
        want_max = p.call(eng, 25, False, False)[0]
        want_d2 = p.call(eng, 25, True, False, us)[0]
        _refused(small, "ALQ_ERR_NOMEM.*peer window too small", lambda: p.call(small, 25, False, True))
        assert p.call(small, 25, False, False)[0] == want_max
        _refused(small, "ALQ_ERR_NOMEM.*peer window too small", lambda: p.call(small, 25, True, True, us))
        assert p.call(small, 25, True, False, us)[0] == want_d2
        assert p.call(eng, 25, False, True)[0] == want_max                  # the group's other context is unaffected
    finally:
        small.close()
