"""BalancingSampler in a ShardGroup of 2 and 3 ranks, on the CPU (gloo): each rank forwards its row_range of the pool,
the embeddings and labels are replicated with all_gather_rows, and the sharded K11 / K12 calls (here: the NumPy twins,
tests/balancing_loop_oracle.py and tests/balancing_table_oracle.py, behind the same host agreement check Engine runs)
must give every rank the reference's picks and the single-process NumPy state.  Mismatched inputs across the ranks raise
AlqError on every rank before any engine work."""
import os
import socket
import sys
import tempfile

import numpy as np
import pytest
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDENS = {"reference_golden_balancing.npz": ("a", "b"), "reference_golden_balancing_loop.npz": ("m", "r"),
           "reference_golden_balancing_table.npz": ("t", "u")}


def load_goldens():
    return {f: dict(np.load(os.path.join(HERE, "golden", f))) for f in GOLDENS}


def seed_of(g, tag):
    return int(g.get(f"{tag}_seed", 11))


def state_key(st):
    return (st[0], np.asarray(st[1]).tolist(), int(st[2]), int(st[3]), float(st[4]))


def make_engine(tag, **kw):
    """K11's twin for the goldens it was made for, K12's (K11 declining) for the 1 000-class ones."""
    from test_balancing_table import TableEngine

    class ShardedTwinEngine(TableEngine):
        """TableEngine with the sharded signature: a call with shard_off first runs the host agreement check of
        Engine._balancing_call (sharding.balancing_agreement), then the twin on the replicated inputs."""

        def __init__(self, **k):
            super().__init__(**k)
            self.shard_offs = []

        def _agree(self, what, args, shard_off):
            from active_learning_b200.sharding import balancing_agreement
            emb, _xn, labels, avail, labeled, c, budget = args
            balancing_agreement(what, tuple(emb.shape), c, budget, shard_off, labels, avail, labeled)
            self.shard_offs.append([int(v) for v in shard_off])

        def balancing_select(self, *args, shard_off=None):
            if shard_off is not None:
                self._agree("alq_balancing_select", args, shard_off)
            return super().balancing_select(*args)

        def balancing_table_select(self, *args, shard_off=None):
            if shard_off is not None:
                self._agree("alq_balancing_table_select", args, shard_off)
            return super().balancing_table_select(*args)

    if tag in ("t", "u"):
        kw.setdefault("centre_floats", 0)
    return ShardedTwinEngine(**kw)


def sampler(g, tag, eng, group=None):
    """The golden's BalancingSampler; its forwards are recorded in s.forwarded (the pool rows asked for)."""
    from test_balancing import balancing_strategy
    s = balancing_strategy(g, tag, engine=eng)
    s._shard_group = group
    s.forwarded = []
    inner = s._forward_pool

    def recording(idxs, *a, **k):
        s.forwarded.append(list(idxs))
        return inner(idxs, *a, **k)

    s._forward_pool = recording
    return s


def run_rounds(g, tag, eng, group=None):
    """Round 1 at the golden budget, then (under --freeze_feature) a round of 5; picks, states and forwards."""
    np.random.seed(seed_of(g, tag))
    s = sampler(g, tag, eng, group)
    idx, cost = s.query(float(g[f"{tag}_budget"]))
    out = {"picks": [int(i) for i in idx], "cost": cost, "state": state_key(np.random.get_state()),
           "forwarded": s.forwarded, "emb": s._bal_cache[0].numpy(), "ys": s._bal_cache[1].numpy()}
    s.update(idx, cost)
    s.forwarded = []
    idx2, _ = s.query(5.0)
    out.update(picks2=[int(i) for i in idx2], forwarded2=s.forwarded, state2=state_key(np.random.get_state()),
               shard_offs=getattr(eng, "shard_offs", None))
    return out


def _worker(rank, world, port, out_path):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from active_learning_b200._lib import AlqError
    from active_learning_b200.sharding import ShardGroup
    golds = load_goldens()
    group = ShardGroup()
    res = {"rank": rank}
    for f, tags in GOLDENS.items():
        for tag in tags:
            res[tag] = run_rounds(golds[f], tag, make_engine(tag), group)
    # both loops decline: the per-step path on the replicated rows
    g = golds["reference_golden_balancing.npz"]
    for tag in ("a", "b"):
        eng = make_engine(tag, centre_floats=0, table_ok=False)
        np.random.seed(11)
        idx, _ = sampler(g, tag, eng, group).query(float(g[f"{tag}_budget"]))
        res[f"{tag}_per_step"] = ([int(i) for i in idx], state_key(np.random.get_state()), eng.declined,
                                  eng.table_declined)
    # inputs that differ across the ranks: AlqError on every rank, the twin never runs
    for what in ("budget", "state"):
        eng = make_engine("m")
        gm = golds["reference_golden_balancing_loop.npz"]
        np.random.seed(seed_of(gm, "m") + (rank if what == "state" else 0))
        s = sampler(gm, "m", eng, group)
        try:
            s.query(float(gm["m_budget"]) + (rank if what == "budget" else 0))
            res[f"mismatch_{what}"] = "no error"
        except AlqError as exc:
            res[f"mismatch_{what}"] = (str(exc), eng.calls, eng.table_calls)
    all_res = [None] * world
    dist.all_gather_object(all_res, res)
    if rank == 0:
        np.save(out_path, np.array(all_res, dtype=object), allow_pickle=True)
    dist.barrier()
    dist.destroy_process_group()


@pytest.fixture(scope="module")
def golds():
    return load_goldens()


@pytest.fixture(scope="module")
def single(golds):
    """The same rounds in one process without a group (the calls and path of today)."""
    return {tag: run_rounds(g, tag, make_engine(tag)) for f, g in golds.items() for tag in GOLDENS[f]}


def run_group(world):
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    out = os.path.join(tempfile.mkdtemp(), "res.npy")
    mp.spawn(_worker, args=(world, port, out), nprocs=world, join=True)
    return list(np.load(out, allow_pickle=True))


@pytest.fixture(scope="module", params=[2, 3])
def group_results(request):
    return request.param, run_group(request.param)


def test_single_process_rounds_are_the_goldens(golds, single):
    for f, tags in GOLDENS.items():
        for tag in tags:
            assert single[tag]["picks"] == golds[f][f"{tag}_picks"].tolist()
            assert single[tag]["shard_offs"] == []                       # no group: no shard_off reaches the engine


def test_every_rank_returns_the_goldens(golds, single, group_results):
    world, results = group_results
    assert [r["rank"] for r in results] == list(range(world))
    for f, tags in GOLDENS.items():
        g = golds[f]
        for tag in tags:
            n = g[f"{tag}_emb"].shape[0]
            bounds = [(r * (n // world) + min(r, n % world), (r + 1) * (n // world) + min(r + 1, n % world))
                      for r in range(world)]
            for res in results:
                got, want = res[tag], single[tag]
                assert got["picks"] == g[f"{tag}_picks"].tolist() and got["cost"] == int(g[f"{tag}_budget"])
                assert got["state"] == want["state"]                     # the NumPy state of the single process
                if f"{tag}_after" in g:
                    np.random.set_state(got["state"])
                    assert np.random.random_sample() == float(g[f"{tag}_after"])
                lo, hi = bounds[res["rank"]]
                assert got["forwarded"] == [list(range(lo, hi))]         # this rank's row_range only
                d = g[f"{tag}_emb"].shape[1]
                assert np.array_equal(got["emb"][:, :d], g[f"{tag}_emb"]) and np.array_equal(got["ys"], g[f"{tag}_ys"])
                assert got["shard_offs"][0] == [b[0] for b in bounds] + [n]
                # second round under --freeze_feature: nothing is forwarded, the same picks as one process
                assert got["forwarded2"] == [] and got["picks2"] == want["picks2"] and got["state2"] == want["state2"]


def test_per_step_path_when_both_loops_decline(golds, group_results):
    from test_balancing_table import _run_loop_twin
    _, results = group_results
    g = golds["reference_golden_balancing.npz"]
    for tag in ("a", "b"):
        _, after = _run_loop_twin(g, tag)
        for res in results:
            picks, state, declined, table_declined = res[f"{tag}_per_step"]
            assert picks == g[f"{tag}_picks"].tolist() and declined == 1 and table_declined == 1
            np.random.set_state(state)
            assert np.random.random_sample() == after


@pytest.mark.parametrize("what,field", [("budget", "budget"), ("state", "MT19937 state")])
def test_mismatched_inputs_raise_on_every_rank(group_results, what, field):
    _, results = group_results
    for res in results:
        msg, calls, table_calls = res[f"mismatch_{what}"]
        assert f"disagree on {field}" in msg and calls == 0 and table_calls == 0
