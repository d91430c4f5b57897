"""K11 and K12 with rows sharded over a peer-memory group (alq_balancing_desc.shard_off_host).

One GPU: a group of one rank (gloo world 1, Engine.comm_init).  The words then live in this GPU's own window, but the
call runs the sharded path -- the ready handshake, epoch-tagged words in the window region shared with the persistent
selection loop, the global segment layout -- and must equal the single-GPU call bit for bit: picks, balancing steps and
NumPy's MT19937 state.  Two or more GPUs (skipped below 2): BalancingSampler in an NCCL group, every rank with the
goldens' picks and the same RNG state."""
import ctypes as C
import os
import socket
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from test_balancing import bgold, masks  # noqa: F401  (fixture)
from test_balancing_loop import _state_equal, lgold  # noqa: F401  (fixture)
from test_gpu_balancing_loop import make_pool
from test_gpu_balancing_table import _golden_case, option, pend_cap, run_twin as run_table_twin

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu

OPTION_FN = {2: "balancing_select", 3: "balancing_table_select"}     # K11, K12


@pytest.fixture(scope="module")
def tgold():
    return dict(np.load(os.path.join(ROOT, "tests", "golden", "reference_golden_balancing_table.npz")))


@pytest.fixture(scope="module")
def eng(tmp_path_factory):
    import torch.distributed as dist
    from active_learning_b200.engine import Engine
    init = tmp_path_factory.mktemp("one_rank_group") / "init"
    dist.init_process_group("gloo", init_method=f"file://{init}", world_size=1, rank=0)
    try:
        e = Engine().comm_init()
        yield e
        e.set_option("balancing_loop", 0)
        e.close()
    finally:
        dist.destroy_process_group()


def device_args(eng, emb, ys, avail, lab, c, budget):
    x = torch.from_numpy(np.ascontiguousarray(emb)).cuda()
    return (x, eng.row_norm2(x), torch.from_numpy(np.asarray(ys, dtype=np.int32)).cuda(),
            torch.from_numpy(avail.astype(np.uint8)).cuda(), torch.from_numpy(lab.astype(np.uint8)).cuda(), c, budget)


def run(eng, args, seed, opt, sharded):
    """-> (picks, balancing steps, NumPy state after) of K11 (opt 2) or K12 (opt 3); shard_off = [0, n] when sharded."""
    kw = {"shard_off": [0, args[0].shape[0]]} if sharded else {}
    np.random.seed(seed)
    with option(eng, opt):
        res = getattr(eng, OPTION_FN[opt])(*args, **kw)
    return res[0].tolist(), res[1], np.random.get_state()


def same_as_unsharded(eng, args, seed, opt):
    one = run(eng, args, seed, opt, False)
    grp = run(eng, args, seed, opt, True)
    assert grp[0] == one[0] and grp[1] == one[1] and _state_equal(grp[2], one[2])
    return grp


GOLDEN_CASES = [("b", "a"), ("b", "b"), ("l", "m"), ("l", "r"), ("t", "t"), ("t", "u")]
# K11 (option 2) runs every golden but the 1 000-class ones, beyond its shared-memory limit; K12 (option 3) runs all
GOLDEN_RUNS = [(src, tag, opt) for src, tag in GOLDEN_CASES for opt in (2, 3) if opt == 3 or src != "t"]


@pytest.mark.parametrize("src,tag,opt", GOLDEN_RUNS)
def test_one_rank_group_equals_single_gpu_on_goldens(eng, bgold, lgold, tgold, src, tag, opt):  # noqa: F811
    g = {"b": bgold, "l": lgold, "t": tgold}[src]
    emb, ys, avail, lb, c, budget = _golden_case(g, tag)
    picks, steps, _ = same_as_unsharded(eng, device_args(eng, emb, ys, avail, lb, c, budget), int(g.get(f"{tag}_seed", 11)), opt)
    assert picks == g[f"{tag}_picks"].tolist() and steps == int(g[f"{tag}_balancing_steps"])


@pytest.mark.parametrize("opt", [2, 3])
@pytest.mark.parametrize("n", [1023, 1024, 1025, 16895, 16896, 16897, 20000])
def test_one_rank_group_segment_edges(eng, n, opt):
    c, d = 5, 32
    emb, ys, avail, lab = make_pool(n, d, c, n, [40, 20, 10, 5, 0])
    for budget in (60, min(n, 400)):
        same_as_unsharded(eng, device_args(eng, emb, ys, avail, lab, c, budget), 3, opt)


def test_one_rank_group_random_run_longer_than_the_pending_list(eng, tgold):
    """The tiled uniform golden of test_gpu_balancing_table.py: runs of random draws longer than K12's pending list."""
    g = tgold
    emb, ys, avail, lb, c, budget = _golden_case(g, "u")
    big = np.ascontiguousarray(np.tile(emb, (1, 341)))
    out = run_table_twin(emb, ys, avail, lb, c, budget, int(g["u_seed"]))
    br = out["branch"]
    longest, cur = 0, 0
    for b in br[br.index(True):]:
        cur = 0 if b else cur + 1
        longest = max(longest, cur)
    assert 1 <= pend_cap(c, big.shape[1]) < longest
    picks, steps, state = same_as_unsharded(eng, device_args(eng, big, ys, avail, lb, c, budget), int(g["u_seed"]), 3)
    assert picks == g["u_picks"].tolist() and steps == int(g["u_balancing_steps"])
    np.random.set_state(state)
    assert np.random.random_sample() == float(g["u_after"])


def imagenet_lt_pool(tgold):
    """115 846 x 2048 rows with ImageNet-LT's class sizes (as test_gpu_balancing_table.py builds them), 10 % labeled."""
    counts = tgold["lt_counts"]
    c, d = 1000, 2048
    rng = np.random.default_rng(7)
    ys = rng.permutation(np.repeat(np.arange(c), counts))
    n = len(ys)
    emb = (rng.standard_normal((c, d), dtype=np.float32) * 0.5)[ys]
    emb += rng.standard_normal((n, d), dtype=np.float32)
    np.maximum(emb, 0, out=emb)
    lab = np.zeros(n, dtype=bool)
    lab[rng.choice(n, size=n // 10, replace=False)] = True
    return emb, ys, ~lab, lab, c


def test_one_rank_group_imagenet_lt_shape(eng, tgold):
    emb, ys, avail, lab, c = imagenet_lt_pool(tgold)
    _, steps, _ = same_as_unsharded(eng, device_args(eng, emb, ys, avail, lab, c, 200), 1, 3)
    assert steps == 200


def test_calls_in_a_row_with_other_group_calls_between(eng):
    """The window region and the ready words are shared with the selection loop and the tail's windows: sharded calls
    separated by a sharded greedy_select and a sharded uncertainty tail keep returning the same result."""
    n, d, c = 20000, 32, 6
    emb, ys, avail, lab = make_pool(n, d, c, 4, [60, 30, 15, 8, 4, 1])
    args = device_args(eng, emb, ys, avail, lab, c, 150)
    want = {opt: run(eng, args, 8, opt, False) for opt in (2, 3)}
    x = torch.rand(3000, 16, device="cuda")
    logits = torch.randn(8192, 12, device="cuda")
    for _ in range(3):
        for opt in (2, 3):
            got = run(eng, args, 8, opt, True)
            assert got[0] == want[opt][0] and got[1] == want[opt][1] and _state_equal(got[2], want[opt][2])
        mind = torch.full((3000,), float("inf"), device="cuda")
        assert eng.greedy_select(x, eng.row_norm2(x), mind, [0, 3000], [7], first_pick=[11],
                                 shard_off=[0, 3000]).tolist()[0] == 11
        _, pos = eng.uncertainty_tail_sharded(logits, 0, 100, 0, 8192, 8192)
        assert torch.equal(pos, eng.select_smallest(eng.score_softmax(logits, 0), 100))
        torch.cuda.synchronize()
        eng.comm_check()


@pytest.mark.parametrize("opt", [2, 3])
def test_launch_count_does_not_depend_on_the_budget(eng, opt):
    n, d, c = 30000, 32, 4
    emb, ys, avail, lab = make_pool(n, d, c, 6, [200, 50, 10, 0])
    counts = []
    for budget in (20, 2000):
        args = device_args(eng, emb, ys, avail, lab, c, budget)
        before = eng.launches
        run(eng, args, 2, opt, True)
        counts.append(eng.launches - before)
    assert counts[0] == counts[1] and counts[0] <= 8


def test_descriptor_of_the_old_size_is_a_single_gpu_call(eng):
    """A descriptor whose struct_size ends before shard_off_host: the field is not read (here it points at offsets that
    a group of one rank would reject) and the call is the single-GPU one."""
    from active_learning_b200 import _lib
    n, d, c, budget = 5000, 16, 4, 40
    emb, ys, avail, lab = make_pool(n, d, c, 3, [50, 20, 5, 1])
    x, xn, labels, av, lb, _, _ = device_args(eng, emb, ys, avail, lab, c, budget)
    want = run(eng, (x, xn, labels, av, lb, c, budget), 5, 2, False)
    np.random.seed(5)
    _, key, pos, _, _ = np.random.get_state()
    key = np.array(key, dtype=np.uint32)
    pos_c, n_picks, n_bal = C.c_int32(int(pos)), C.c_int64(0), C.c_int64(0)
    bad_off = np.array([0, n // 2, n], dtype=np.int32)
    picks = torch.empty(budget, dtype=torch.int32, device="cuda")
    desc = _lib.BalancingDesc()
    desc.struct_size = _lib.BalancingDesc.shard_off_host.offset
    desc.x, desc.ldx, desc.d = x.data_ptr(), d, d
    desc.xn, desc.labels, desc.avail, desc.labeled = xn.data_ptr(), labels.data_ptr(), av.data_ptr(), lb.data_ptr()
    desc.n, desc.c, desc.budget = n, c, budget
    desc.mt_key_host, desc.mt_pos_host = key.ctypes.data, C.addressof(pos_c)
    desc.picks, desc.n_picks_host, desc.n_balancing_host = picks.data_ptr(), C.addressof(n_picks), C.addressof(n_bal)
    desc.shard_off_host = bad_off.ctypes.data
    with option(eng, 2):
        eng._check(eng.lib.alq_balancing_select(eng._h, C.byref(desc), eng._stream()), "alq_balancing_select")
    assert n_picks.value == budget and picks.cpu().tolist() == want[0] and n_bal.value == want[1]
    assert np.array_equal(key, want[2][1]) and int(pos_c.value) == want[2][2]


def test_sharded_call_needs_a_group_and_valid_offsets(eng):
    from active_learning_b200.engine import AlqError
    n, d, c = 2000, 16, 3
    emb, ys, avail, lab = make_pool(n, d, c, 2, [20, 10, 0])
    args = device_args(eng, emb, ys, avail, lab, c, 10)
    with pytest.raises(AlqError, match="offsets"):
        eng.balancing_select(*args, shard_off=[0, n // 2, n])        # a group of one rank takes two offsets
    with pytest.raises(AlqError, match="shard_off must run from 0 to n"):
        eng.balancing_select(*args, shard_off=[0, n - 1])


# ---- two or more GPUs ----------------------------------------------------------------------------------------------
def _worker(rank, world, port, out_path):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    import torch.distributed as dist
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from test_balancing import balancing_strategy
    from active_learning_b200.engine import Engine
    from active_learning_b200.sharding import ShardGroup
    eng = Engine(rank).comm_init()
    group = ShardGroup()
    golds = {src: dict(np.load(os.path.join(ROOT, "tests", "golden", f))) for src, f in
             (("b", "reference_golden_balancing.npz"), ("l", "reference_golden_balancing_loop.npz"),
              ("t", "reference_golden_balancing_table.npz"))}
    res = {}
    for src, tag, opt in GOLDEN_RUNS + [(src, tag, 0) for src, tag in GOLDEN_CASES]:
        g = golds[src]
        s = balancing_strategy(g, tag, engine=eng)
        s._shard_group = group
        np.random.seed(int(g.get(f"{tag}_seed", 11)))
        eng.set_option("balancing_loop", opt)
        idx, _ = s.query(float(g[f"{tag}_budget"]))
        eng.set_option("balancing_loop", 0)
        _, key, pos, _, _ = np.random.get_state()
        res[(tag, opt)] = ([int(i) for i in idx], np.asarray(key).tolist(), int(pos))
    # ImageNet-LT's shape: the sharded K12 call against this GPU's unsharded one
    emb, ys, avail, lab, c = imagenet_lt_pool(golds["t"])
    args = device_args(eng, emb, ys, avail, lab, c, 200)
    n = emb.shape[0]
    one = run(eng, args, 1, 3, False)
    np.random.seed(1)
    with option(eng, 3):
        grp = eng.balancing_table_select(*args, shard_off=[group.row_range(n, r)[0] for r in range(world)] + [n])
    res["lt"] = (grp[0].tolist() == one[0], grp[1] == one[1], _state_equal(np.random.get_state(), one[2]), grp[0].tolist())
    all_res = [None] * world
    dist.all_gather_object(all_res, res)
    if rank == 0:
        np.save(out_path, np.array(all_res, dtype=object), allow_pickle=True)
    dist.barrier()
    eng.close()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_sampler_returns_the_goldens_on_every_rank(bgold, lgold, tgold):  # noqa: F811
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    out = os.path.join(tempfile.mkdtemp(), "res.npy")
    mp.spawn(_worker, args=(2, port, out), nprocs=2, join=True)
    results = list(np.load(out, allow_pickle=True))
    golds = {"b": bgold, "l": lgold, "t": tgold}
    for src, tag, opt in GOLDEN_RUNS + [(src, tag, 0) for src, tag in GOLDEN_CASES]:
        got = [r[(tag, opt)] for r in results]
        assert all(x == got[0] for x in got[1:])                  # picks and MT19937 state identical on every rank
        assert got[0][0] == golds[src][f"{tag}_picks"].tolist()
    for r in results:
        assert r["lt"][:3] == (True, True, True) and r["lt"][3] == results[0]["lt"][3]
