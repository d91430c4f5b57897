"""ProbCoverSampler without a GPU: the oracle's greedy against the authors' loop, the tensor-core screen's bound against
fp64 truth, and the sampler's host logic (RNG draws, budget clamp, cache, pickling) through a fake engine built on the
oracle."""
import os
import pickle

import numpy as np
import pytest
import torch

import probcover_oracle as P
from helpers import OracleEngine, make_strategy


def _edges(row_ptr, cols):
    x = np.repeat(np.arange(len(row_ptr) - 1), np.diff(row_ptr))
    return x.astype(np.int64), cols.astype(np.int64)


def test_oracle_greedy_equals_the_authors_loop_on_random_graphs():
    rng = np.random.default_rng(0)
    for trial in range(40):
        n = int(rng.integers(1, 300))
        d = int(rng.integers(2, 12))
        x = rng.normal(size=(n, d)).astype(np.float32)
        if trial % 4 == 1:
            x[rng.integers(0, n, n // 3)] = x[0]                      # duplicated rows: degree ties
        xh = P.normalize(x)
        delta = float(rng.uniform(0.2, 1.6))
        row_ptr, cols = P.graph(xh, delta)
        lab = rng.random(n) < (0.0 if trial % 3 == 0 else 0.1)
        ex, ey = _edges(row_ptr, cols)
        mine = P.greedy(row_ptr, cols, lab, n)
        theirs = P.authors_greedy(ex, ey, n, np.flatnonzero(lab), n)
        assert mine.tolist() == theirs.tolist()
        # the graph is symmetric, every row holds itself, and the columns are ascending
        assert set(zip(ex.tolist(), ey.tolist())) == set(zip(ey.tolist(), ex.tolist()))
        for r in range(n):
            seg = cols[row_ptr[r]:row_ptr[r + 1]]
            assert r in seg and (np.diff(seg) > 0).all()


def test_normalize_is_the_stated_order_and_keeps_zero_rows():
    rng = np.random.default_rng(1)
    x = rng.normal(size=(50, 70)).astype(np.float32) * np.float32(1e3)
    x[3] = 0
    xh = P.normalize(x)
    assert (xh[3] == 0).all()
    assert np.allclose(np.linalg.norm(xh.astype(np.float64), axis=1)[np.arange(50) != 3], 1.0, atol=1e-6)
    # padding with zero columns changes nothing
    xp = np.zeros((50, 96), dtype=np.float32)
    xp[:, :70] = x
    assert (P.normalize(xp)[:, :70] == xh).all()


def _adversarial_rows(rng, d):
    rows = [np.ones(d), -np.ones(d), rng.normal(size=d), np.exp(rng.normal(0, 4, d)) * rng.choice([-1, 1], d)]
    spike = np.full(d, 1e-4)
    spike[0] = 1.0
    rows.append(spike)
    # entries on TF32 rounding midpoints (the largest split error)
    mid = (rng.integers(1 << 22, 1 << 23, d).astype(np.uint32) | np.uint32(0x1000)) & ~np.uint32(0xFFF)
    rows.append(mid.view(np.float32) * np.float32(1e-6))
    rows.append(np.abs(rng.normal(size=d)))
    x = np.stack(rows).astype(np.float32)
    near = x + (rng.normal(size=x.shape) * 1e-4).astype(np.float32)    # near-duplicates: d2 next to 0
    return P.normalize(np.concatenate([x, near, -x]))


@pytest.mark.parametrize("d", [4, 64, 2048])
def test_screen_bound_holds_against_fp64_truth_on_adversarial_rows(d):
    rng = np.random.default_rng(d)
    xh = _adversarial_rows(rng, d)
    m = xh.shape[0]
    i, j = np.triu_indices(m)
    x64 = xh.astype(np.float64)
    nrm = (x64 * x64).sum(axis=1)
    truth = (x64[i] * x64[j]).sum(axis=1)
    bound = P.screen_bound(d, nrm[i], nrm[j])
    for adder in ("nearest", "zero", "align"):
        g = P.emulate_3xtf32(xh[i], xh[j], adder=adder).astype(np.float64)
        assert (np.abs(g - truth) <= bound).all(), (adder, np.max(np.abs(g - truth) / bound))
        # every certified decision is the exact one, for radii placed on the pairs' own distances
        exact = P.exact_d2(xh[i], xh[j])
        n2 = P.nrm2(xh)
        for delta in np.sqrt(np.clip(exact[::7], 1e-12, None)).tolist() + [0.5, 1.0, 1.9]:
            dec = P.screen_decide(d, n2[i], n2[j], g, delta)
            truth_edge = np.sqrt(exact) < delta
            assert truth_edge[dec == P.EDGE].all() and not truth_edge[dec == P.NONE].any()


@pytest.mark.parametrize("d", [4, 28, 36, 64, 520, 2048])
def test_screen_bound_holds_on_the_bound_families_under_every_adder_model(d):
    """The rows the H100 probe (test_gpu_tf32_bound.py) measures, every pair within and across families, under the
    three adder models; the align-and-truncate adder keeps 24 bits.  An align adder of 21 bits breaks E on these rows
    from d = 28 on, so they are adversarial enough to tell the two apart."""
    fam = P.bound_families(np.random.default_rng(100 + d), d)
    xh = np.concatenate(list(fam.values()))
    i, j = np.triu_indices(len(xh))
    truth = P.exact_dots(xh[i], xh[j])
    nrm = P.nrm2(xh)
    bound = P.screen_bound(d, nrm[i], nrm[j])

    def worst(adder, bits=24):
        return np.max(np.abs(P.emulate_3xtf32(xh[i], xh[j], adder=adder, bits=bits).astype(np.float64) - truth) / bound)

    for adder in ("nearest", "zero", "align"):
        assert worst(adder) <= 1.0, (adder, d, worst(adder))
    if d >= 28:
        assert worst("align", bits=21) > 1.0


def test_the_adder_models_are_exact_on_tf32_integers_and_differ_elsewhere():
    rng = np.random.default_rng(4)
    a = rng.integers(-8, 9, size=(64, 520)).astype(np.float32)
    b = rng.integers(-8, 9, size=(64, 520)).astype(np.float32)
    want = (a.astype(np.float64) * b).sum(axis=1)
    for adder in ("nearest", "zero", "align"):
        assert (P.emulate_3xtf32(a, b, adder=adder).astype(np.float64) == want).all()
    fam = P.bound_families(np.random.default_rng(5), 2048)["full_mantissa"]
    g = {ad: P.emulate_3xtf32(fam, fam[::-1], adder=ad) for ad in ("nearest", "zero", "align")}
    assert (g["align"] != g["nearest"]).any() and (g["align"] != g["zero"]).any()
    assert (P.emulate_3xtf32(fam, fam[::-1], adder="align", bits=21) != g["align"]).any()


# ---- the sampler's host logic ------------------------------------------------------------------------------------------
class ProbCoverEngine(OracleEngine):
    """The oracle engine plus K13 / K14 by the NumPy statement; counts the graph builds."""

    def __init__(self):
        self.graphs = 0

    def probcover_graph(self, x, delta):
        self.graphs += 1
        row_ptr, cols = P.graph(P.normalize(x.numpy()), float(delta))
        return torch.from_numpy(row_ptr), torch.from_numpy(cols), 0

    def probcover_select(self, row_ptr, cols, labeled, budget):
        picks = P.greedy(row_ptr.numpy(), cols.numpy(), labeled.numpy().astype(bool), budget)
        return picks, len(picks)


def _pool(n=160, d=6, seed=3):
    rng = np.random.default_rng(seed)
    emb = torch.from_numpy(rng.normal(size=(n, d)).astype(np.float32))
    logits = torch.zeros(n, 4)
    eval_idxs = rng.choice(n, 12, replace=False)
    rest = np.setdiff1d(np.arange(n), eval_idxs)
    labeled = rng.choice(rest, 9, replace=False)
    return emb, logits, eval_idxs, labeled


def _expected(s, emb, budget, delta):
    """What the query returns and leaves in NumPy's RNG, replayed from the same state: the two shuffles, the oracle."""
    union = np.asarray(s.get_idxs_for_coreset(), dtype=np.int64)
    is_lab = s.already_labeled_idxs(boolean=True)[union]
    avail = s.available_query_idxs(boolean=True)[union]
    pos = P.query_positions(emb.numpy()[union], is_lab, avail, budget, delta)
    return union[pos].tolist()


@pytest.mark.parametrize("delta,budget", [(0.6, 7), (0.9, 25), (3.0, 11), (0.6, 10 ** 6), (0.05, 30)])
def test_query_equals_the_oracle_with_numpys_draws(delta, budget):
    emb, logits, ev, lab = _pool()
    eng = ProbCoverEngine()
    s = make_strategy("ProbCoverSampler", logits, emb, ev, lab, 32, engine=eng, delta=delta)
    np.random.seed(11)
    got, k = s.query(budget)
    state = np.random.get_state()
    np.random.seed(11)
    want = _expected(s, emb, budget, delta)
    assert got == want and k == len(want)
    assert k == min(budget, int(s.available_query_idxs(boolean=True).sum()))
    assert len(set(got)) == k and not s.idxs_lb[got].any() and not np.isin(got, ev).any()
    after = np.random.get_state()
    assert state[2] == after[2] and (state[1] == after[1]).all()


def test_zero_budget_returns_nothing_and_draws_only_the_pool():
    emb, logits, ev, lab = _pool()
    eng = ProbCoverEngine()
    s = make_strategy("ProbCoverSampler", logits, emb, ev, lab, 32, engine=eng, delta=0.7)
    np.random.seed(5)
    assert s.query(0) == ([], 0)
    state = np.random.get_state()
    np.random.seed(5)
    s.get_idxs_for_coreset()
    assert (np.random.get_state()[1] == state[1]).all() and eng.graphs == 0


def test_delta_is_required_finite_and_positive():
    emb, logits, ev, lab = _pool()
    for bad in (None, 0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            make_strategy("ProbCoverSampler", logits, emb, ev, lab, 32, engine=ProbCoverEngine(), delta=bad)


def test_the_graph_is_cached_across_rounds_and_rebuilt_when_it_must_be():
    emb, logits, ev, lab = _pool()
    eng = ProbCoverEngine()
    s = make_strategy("ProbCoverSampler", logits, emb, ev, lab, 32, engine=eng, delta=0.8)
    np.random.seed(2)
    for rnd in range(3):
        np.random.seed(20 + rnd)
        state = np.random.get_state()
        got, k = s.query(6)
        np.random.set_state(state)
        assert got == _expected(s, emb, 6, 0.8)
        s.update(got, k)
        s.round += 1
    assert eng.graphs == 1
    s.delta = 0.5                                                     # another radius: rebuilt, then cached again
    s.query(4)
    s.query(4)
    assert eng.graphs == 2
    blob = pickle.dumps(s)
    assert b"_pc_cache" not in blob or pickle.loads(blob).__dict__.get("_pc_cache") is None
    s2 = pickle.loads(blob)
    s2.set_engine(eng)
    s2.query(4)
    assert eng.graphs == 3
    for kw in ({"subset_unlabeled": 100}, {"freeze_feature": False}):
        e2 = ProbCoverEngine()
        t = make_strategy("ProbCoverSampler", logits, emb, ev, lab, 32, engine=e2, delta=0.8, **kw)
        t.query(3)
        t.query(3)
        assert e2.graphs == 2


def _one_query():
    emb, logits, ev, lab = _pool()
    s = make_strategy("ProbCoverSampler", logits, emb, ev, lab, 32, engine=ProbCoverEngine(), delta=0.7)
    return s


def _worker(rank, world, port, out_path):
    import os
    import sys
    import torch.distributed as dist
    here = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, os.path.dirname(here))
    sys.path.insert(0, here)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from active_learning_b200.sharding import ShardGroup
    from test_probcover import _one_query
    s = _one_query()
    s._shard_group = ShardGroup()
    np.random.seed(9)
    res = s.query(40)
    all_res = [None] * world
    dist.all_gather_object(all_res, res)
    if rank == 0:
        np.save(out_path, np.array(all_res, dtype=object), allow_pickle=True)
    dist.barrier()
    dist.destroy_process_group()


def test_world_size_two_returns_the_one_rank_picks_on_every_rank():
    import os
    import socket
    import tempfile
    import torch.multiprocessing as mp
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    out = os.path.join(tempfile.mkdtemp(), "res.npy")
    mp.spawn(_worker, args=(2, port, out), nprocs=2, join=True)
    np.random.seed(9)
    want = _one_query().query(40)
    for got in np.load(out, allow_pickle=True):
        assert tuple(got) == tuple(want)
