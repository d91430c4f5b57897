"""BalancedRandomSampler without a GPU: the oracle (tests/balanced_random_oracle.py) against the reference's goldens
(tests/golden/make_golden_balanced_random.py), the closed-form per-class budgets against the reference's loop, and the
sampler's host logic -- RNG draws, order, types, the documented deviations, rounds, dispatch, pickling, a gloo group of
two ranks -- with a CPU engine that implements K10's two calls in NumPy."""
import os
import pickle
import socket
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import balanced_random_oracle as BR
from helpers import FakeExperiment, OracleEngine

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_balanced_random as G  # noqa: E402

TAGS = list(G.FIXTURES)


def load_gold():
    return dict(np.load(os.path.join(HERE, "golden", "reference_golden_balanced_random.npz")))


@pytest.fixture(scope="module")
def bgold():
    return load_gold()


def usable(gold, tag):
    """The `ties` fixture holds only where this host's np.argsort orders the tied counts as the generator's did."""
    if tag != "ties":
        return True
    ys, ev, lab = gold[f"{tag}_labels"], gold[f"{tag}_eval"], gold[f"{tag}_labeled"]
    counts = np.bincount(ys[G.avail_mask(len(ys), ev, lab)], minlength=G.FIXTURES[tag][0]).astype(np.float64)
    return np.array_equal(np.argsort(counts), gold[f"{tag}_argsort"])


def skip_unusable(gold, tag):
    if not usable(gold, tag):
        pytest.skip("np.argsort on this host orders the tied class counts differently from the host that generated the "
                    "'ties' golden, so the reference itself would pick other classes here")


class ClassOracleEngine(OracleEngine):
    """The CPU engine stub with K10 in NumPy: same contract as Engine.class_counts / class_pick."""

    def __init__(self):
        self.launches = 0

    def class_counts(self, labels, avail, num_classes):
        from active_learning_b200._lib import AlqError
        y, a = labels.numpy().astype(np.int64), avail.numpy().astype(bool)
        bad = np.flatnonzero(a & ((y < 0) | (y >= num_classes)))
        if bad.size:
            raise AlqError(f"alq_class_counts: ALQ_ERR_INVALID: available row {bad[0]} has label {y[bad[0]]}")
        self.launches += 2
        return torch.from_numpy(np.bincount(y[a], minlength=num_classes).astype(np.int32))

    def class_pick(self, labels, avail, k, perm):
        y, a = labels.numpy(), avail.numpy().astype(bool)
        k, perm = np.asarray(k, dtype=np.int64), np.asarray(perm, dtype=np.int64)
        out, at = [], 0
        for c in range(len(k)):
            rows = np.flatnonzero((y == c) & a)
            out += [int(rows[r]) if r < len(rows) else -1 for r in perm[at:at + k[c]]]
            at += k[c]
        self.launches += 4
        return torch.tensor(out, dtype=torch.int32)


def make_sampler(ys, c, ev, lab, engine=None, targets=None, base=None):
    ds = G.LabeledPool(ys, c)
    if targets is not None:
        ds.targets = targets
    if base is None:
        from active_learning_b200.query_strategies.get_strategy import get_strategy
        base = get_strategy("BalancedRandomSampler")
    s = base(ds, ds, None, {"loader_te_args": {"batch_size": 8, "num_workers": 0}}, np.asarray(ev, dtype=np.int64),
             FakeExperiment(), None, ckpt_path=tempfile.mkdtemp(prefix="alq_test_"), exp_name="t")
    s.set_engine(ClassOracleEngine() if engine is None else engine)
    if len(lab):
        s.update(np.asarray(lab), len(lab))
    return s


def fixture_sampler(gold, tag, engine=None, **kw):
    c = G.FIXTURES[tag][0]
    return make_sampler(gold[f"{tag}_labels"], c, gold[f"{tag}_eval"], gold[f"{tag}_labeled"], engine, **kw)


def golden_query(gold, s, tag):
    """One query under the golden seeds: (picks, cost, torch digest, NumPy state unchanged)."""
    np.random.seed(int(gold["np_seed"]))
    torch.manual_seed(int(gold["torch_seed"]))
    before = BR.np_rng_digest()
    idx, cost = s.query(float(gold[f"{tag}_budget"]))
    return idx, cost, BR.torch_rng_digest(), BR.np_rng_digest() == before


def assert_golden(gold, tag, idx, cost, torch_d, np_same):
    assert isinstance(idx, list) and all(type(v) is int for v in idx) and type(cost) is int
    assert idx == gold[f"{tag}_picks"].tolist() and cost == int(gold[f"{tag}_cost"])
    assert torch_d == str(gold[f"{tag}_torch_digest"]) and np_same == bool(gold[f"{tag}_np_unchanged"])


def test_fixtures_cover_the_cases(bgold):
    for tag, want in (("balanced", lambda t, o, b, c: o == 0 and t == b // c),
                      ("longtail", lambda t, o, b, c: o > 0 and t > b // c),
                      ("ties", lambda t, o, b, c: o > 0)):
        c, budget = G.FIXTURES[tag][0], int(bgold[f"{tag}_budget"])
        ys, ev, lab = bgold[f"{tag}_labels"], bgold[f"{tag}_eval"], bgold[f"{tag}_labeled"]
        counts = np.bincount(ys[G.avail_mask(len(ys), ev, lab)], minlength=c)
        _k, t, o, _ = BR.reference_budgets(counts, budget, c)
        assert want(t, o, budget, c), tag
    lt = bgold["longtail_labels"]
    avail = G.avail_mask(len(lt), bgold["longtail_eval"], bgold["longtail_labeled"])
    assert (np.bincount(lt, minlength=100) == 0).any() and ((np.bincount(lt, minlength=100) > 0) &
                                                            (np.bincount(lt[avail], minlength=100) == 0)).any()
    assert int(bgold["all_cost"]) < int(bgold["all_budget"]) and int(bgold["zero_cost"]) == 0


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_replays_the_reference_goldens(bgold, tag):
    skip_unusable(bgold, tag)
    c = G.FIXTURES[tag][0]
    ys, ev, lab = bgold[f"{tag}_labels"], bgold[f"{tag}_eval"], bgold[f"{tag}_labeled"]
    torch.manual_seed(int(bgold["torch_seed"]))
    idx, cost = BR.balanced_random_query([int(v) for v in ys], G.avail_mask(len(ys), ev, lab), c,
                                         float(bgold[f"{tag}_budget"]))
    assert idx == bgold[f"{tag}_picks"].tolist() and cost == int(bgold[f"{tag}_cost"])
    assert BR.torch_rng_digest() == str(bgold[f"{tag}_torch_digest"])


def test_closed_form_budgets_equal_the_reference_loop():
    from active_learning_b200.query_strategies.balanced_random import balanced_class_budgets
    rng = np.random.default_rng(0)
    seen = set()
    for it in range(12000):
        c = 1 if it % 10 == 0 else int(rng.integers(1, 60))
        kind = it % 4
        if kind == 0:                               # heavy ties: few distinct values
            counts = rng.choice(rng.integers(0, 12, 3), size=c)
        elif kind == 1:                             # long tail with zeros
            counts = np.floor(rng.integers(1, 200) / np.arange(1, c + 1) ** rng.uniform(0.5, 2)).astype(np.int64)
            counts[rng.random(c) < 0.2] = 0
        else:
            counts = rng.integers(0, rng.integers(1, 40), c)
        total = int(counts.sum())
        budget = (0, total, int(rng.integers(0, total + 1)), int(rng.integers(0, total + 1)))[it % 4]
        seen.add((c == 1, budget == 0, budget == total and total > 0, bool((counts == 0).any())))
        ref = BR.reference_budgets(counts.astype(np.float64), budget, c)[0]
        got = balanced_class_budgets(counts, budget, c)
        assert got.dtype == np.int32 and np.array_equal(got, ref), (counts.tolist(), budget)
    assert {(True, True), (True, False)} <= {s[:2] for s in seen} and any(s[2] for s in seen) and any(s[3] for s in seen)
    with pytest.raises(ValueError):
        balanced_class_budgets([1, 2], 4, 2)        # more than the available rows: the reference never terminates
    with pytest.raises(ValueError):
        balanced_class_budgets([1, 2], -1, 2)


@pytest.mark.parametrize("tag", TAGS)
def test_sampler_replays_the_reference_goldens(bgold, tag):
    skip_unusable(bgold, tag)
    s = fixture_sampler(bgold, tag)
    assert_golden(bgold, tag, *golden_query(bgold, s, tag))


@pytest.mark.parametrize("form", ["ndarray", "tensor"])
def test_targets_as_array_or_tensor(bgold, form):
    ys = bgold["c1000_labels"]
    targets = ys.copy() if form == "ndarray" else torch.from_numpy(ys.copy())
    s = fixture_sampler(bgold, "c1000", targets=targets)
    assert_golden(bgold, "c1000", *golden_query(bgold, s, "c1000"))


def test_one_row_class_is_picked():
    """The reference raises IndexError here (`.squeeze()` of a single row); randperm(1) draws nothing."""
    ys = np.array([0] * 10 + [1] + [2] * 5)
    s = make_sampler(ys, 3, [], [])
    torch.manual_seed(3)
    idx, cost = s.query(6.0)
    d = BR.torch_rng_digest()
    torch.manual_seed(3)
    assert (idx, cost) == BR.balanced_random_query(ys.tolist(), np.ones(len(ys), dtype=bool), 3, 6.0)
    assert BR.torch_rng_digest() == d and 10 in idx and cost == 6
    g = torch.get_rng_state()
    torch.randperm(1)
    assert torch.equal(g, torch.get_rng_state())


@pytest.mark.parametrize("bad", [3, 1000, -1])
def test_out_of_range_label_raises_before_any_draw(bad):
    ys = np.array([0, 1, 2] * 6)
    ys[7] = bad
    s = make_sampler(ys, 3, [], [])
    torch.manual_seed(5)
    np.random.seed(5)
    t0, n0 = BR.torch_rng_digest(), BR.np_rng_digest()
    with pytest.raises(IndexError, match=f"row 7 .*label {bad}"):
        s.query(6.0)
    assert BR.torch_rng_digest() == t0 and BR.np_rng_digest() == n0
    # the same label on a row that is not available is never looked at
    s.update(np.array([7]), 1)
    idx, cost = s.query(6.0)
    assert cost == 6 and 7 not in idx


def test_negative_and_zero_budget_return_nothing(bgold):
    s = fixture_sampler(bgold, "balanced")
    torch.manual_seed(0)
    t0 = BR.torch_rng_digest()
    assert s.query(-5.0) == ([], 0) and s.query(0.0) == ([], 0) and s.query(0.7) == ([], 0)
    assert BR.torch_rng_digest() == t0 and s.get_engine().launches == 0


def test_three_rounds_equal_the_oracle(bgold):
    c = 100
    ys, ev, lab = bgold["longtail_labels"], bgold["longtail_eval"], bgold["longtail_labeled"]
    s = make_sampler(ys, c, ev, lab)
    mask = G.avail_mask(len(ys), ev, lab)
    torch.manual_seed(11)
    for budget in (300.0, 450.0, 10000.0):
        st = torch.get_rng_state()
        idx, cost = s.query(budget)
        after = torch.get_rng_state()
        torch.set_rng_state(st)
        assert (idx, cost) == BR.balanced_random_query(ys.tolist(), mask, c, budget)
        assert torch.equal(after, torch.get_rng_state())
        s.update(np.array(idx), cost)
        mask[idx] = False
    assert not mask.any() and not s.available_query_idxs(boolean=True).any()


def test_dispatch_and_drop_in_binding(bgold):
    from active_learning_b200.integration import make_drop_in
    from active_learning_b200.query_strategies.balanced_random import BalancedRandomQuery
    from active_learning_b200.query_strategies.get_strategy import ACCELERATED, NOT_ON_THIS_PATH, get_strategy
    from active_learning_b200.query_strategies.strategy import Strategy
    assert "BalancedRandomSampler" in ACCELERATED and NOT_ON_THIS_PATH == ()
    assert get_strategy("BalancedRandomSampler").__name__ == "BalancedRandomSampler"
    cls = make_drop_in(Strategy)["BalancedRandomSampler"]
    assert cls.__bases__ == (BalancedRandomQuery, Strategy)
    for tag in ("balanced", "longtail"):
        s = fixture_sampler(bgold, tag, base=cls)
        assert_golden(bgold, tag, *golden_query(bgold, s, tag))


def test_pickling_round_trip(bgold):
    s = fixture_sampler(bgold, "c1000")
    t = pickle.loads(pickle.dumps(s))
    assert t._engine is None
    t.set_engine(ClassOracleEngine())
    assert_golden(bgold, "c1000", *golden_query(bgold, t, "c1000"))


def _worker(rank, world, port, out_path):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from active_learning_b200.sharding import ShardGroup
    from test_balanced_random import fixture_sampler, golden_query, load_gold
    gold = load_gold()
    group = ShardGroup()
    res = {}
    for tag in ("balanced", "longtail", "c1000"):
        s = fixture_sampler(gold, tag)
        s._shard_group = group
        res[tag] = golden_query(gold, s, tag)
    all_res = [None] * world
    dist.all_gather_object(all_res, res)
    if rank == 0:
        np.save(out_path, np.array(all_res, dtype=object), allow_pickle=True)
    dist.barrier()
    dist.destroy_process_group()


def test_world_size_two_returns_the_same_list_on_every_rank(bgold):
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    out = os.path.join(tempfile.mkdtemp(), "res.npy")
    mp.spawn(_worker, args=(2, port, out), nprocs=2, join=True)
    for res in np.load(out, allow_pickle=True):          # every rank
        for tag, got in res.items():
            assert_golden(bgold, tag, *got)
