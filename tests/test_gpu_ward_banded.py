"""K8 over the banded layout (alq_ward_nn_chain_banded) on the H100, the band memory calls (alq_band_alloc / open /
close / free), and ShardGroup.ward_labels's distributed placement.

The banded walk must give the condensed walk's merge list bit for bit (and the NumPy oracle's, where it runs) for every
band plan of up to 8 bands, with the bands in separate allocations.  The distributed placement runs in a group of one
rank, in a gloo group of two processes on this one GPU (process 0's K8 reads process 1's band through a real CUDA IPC
mapping), and, on two or more GPUs, in an NCCL group (skipped below two GPUs)."""
import ctypes
import os
import socket
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import ward_oracle as W

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
TAGS = ("f", "s", "t", "b")


@pytest.fixture(scope="module")
def eng(tmp_path_factory):
    from helpers import one_rank_engine
    with one_rank_engine(tmp_path_factory.mktemp("ward_banded_one_rank")) as e:
        yield e


@pytest.fixture(scope="module")
def group(eng):
    from active_learning_b200.sharding import ShardGroup
    return ShardGroup()


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(os.path.join(HERE, "golden", "reference_golden_margin_clustering.npz")))


def _rows(n, d, seed):
    rng = np.random.default_rng(seed)
    return np.maximum(rng.standard_normal((n, d)), 0).astype(np.float32)


def _bands(eng, vec, plan, n, separate=True):
    """The bands of `plan` as copies of the condensed vector's slices: each in an allocation of its own (band_alloc),
    or as torch tensors; None for a band without pairs.  Returns (bands for nn_chain_banded, owned WardBands)."""
    from active_learning_b200.sharding import band_pairs
    parts, owned = [], []
    for lo, hi in zip(plan, plan[1:]):
        m, at = band_pairs(n, lo, hi), band_pairs(n, 0, lo)
        if not m:
            parts.append(None)
            continue
        if separate:
            b = eng.band_alloc(8 * m)
            b.tensor()[:m].copy_(vec[at:at + m])
            owned.append(b)
            parts.append(b)
        else:
            parts.append(vec[at:at + m].clone())
    return parts, owned


def _chain(eng, vec, n):
    xy, md = eng.nn_chain(vec.clone(), n)
    return xy.cpu().numpy(), md.cpu().numpy()


def _banded(eng, vec, plan, n, separate=True):
    parts, owned = _bands(eng, vec, plan, n, separate)
    try:
        xy, md = eng.nn_chain_banded(plan, parts, n)
        return xy.cpu().numpy(), md.cpu().numpy()
    finally:
        torch.cuda.synchronize()
        for b in owned:
            b.release()


@pytest.mark.parametrize("n", [2, 3, 63, 64, 65, 129, 4097])
def test_banded_k8_equals_condensed_k8_and_the_oracle_for_every_plan(eng, n):
    from test_gpu_margin_clustering_sharded import _splits
    x = _rows(n, 7, n)
    vec = eng.pdist(torch.from_numpy(x).cuda(), condensed=True)
    want_xy, want_md = _chain(eng, vec, n)
    oxy, omd, _ = W.ward_nn_chain(W.pdist_square(x))
    assert np.array_equal(want_xy, oxy) and np.array_equal(want_md, omd)
    plans = [p for p in _splits(n) if len(p) - 1 <= 8]
    assert len(plans) >= 10
    for k, plan in enumerate(plans):
        xy, md = _banded(eng, vec, plan, n, separate=k % 2 == 0)
        assert np.array_equal(xy, want_xy) and np.array_equal(md.view(np.int64), want_md.view(np.int64)), plan


def test_ward_bands_plans_at_12000_rows_of_2048(eng):
    from active_learning_b200.sharding import ward_bands
    n = 12000
    x = torch.relu(torch.randn(n, 2048, device="cuda", generator=torch.Generator(device="cuda").manual_seed(12)))
    vec = eng.pdist(x, condensed=True)
    want_xy, want_md = _chain(eng, vec, n)
    for g in range(2, 9):
        xy, md = _banded(eng, vec, ward_bands(n, g), n)
        assert np.array_equal(xy, want_xy) and np.array_equal(md.view(np.int64), want_md.view(np.int64)), g


def test_three_bands_past_2_31_entries_at_70000_rows(eng):
    """n (n - 1) / 2 = 2.45e9 > 2^31 entries: three bands of ward_bands(n, 3) in allocations of their own (19.6 GB in
    all) against the condensed walk over the whole vector."""
    from active_learning_b200.sharding import band_pairs, ward_bands
    n = 70000
    if eng._ward_free_bytes() < 2 * 4 * n * (n - 1) + (2 << 30):
        pytest.skip(f"needs {2 * 4 * n * (n - 1)} bytes of free device memory")
    x = torch.from_numpy(_rows(n, 64, n)).cuda()
    b = ward_bands(n, 3)
    assert band_pairs(n, 0, b[2]) < 1 << 31 < n * (n - 1) // 2
    vec = eng.pdist(x, condensed=True)
    parts, owned = _bands(eng, vec, b, n)
    try:
        want_xy, want_md = (t.cpu().numpy() for t in eng.nn_chain(vec, n))
        del vec
        torch.cuda.empty_cache()
        xy, md = (t.cpu().numpy() for t in eng.nn_chain_banded(b, parts, n))
    finally:
        torch.cuda.synchronize()
        for p in owned:
            p.release()
    assert np.array_equal(xy, want_xy) and np.array_equal(md.view(np.int64), want_md.view(np.int64))


def test_a_non_finite_band_gives_numeric_and_the_context_stays_usable(eng):
    from active_learning_b200._lib import AlqError
    n = 300
    x = torch.from_numpy(_rows(n, 5, 3)).cuda()
    vec = eng.pdist(x, condensed=True)
    bad = vec.clone()
    from active_learning_b200.sharding import band_pairs
    row = 17                                              # row 17's distances to every other row: NaN
    for j in range(n):
        if j != row:
            i, k = min(j, row), max(j, row)
            bad[band_pairs(n, 0, i) + (k - i - 1)] = float("nan")
    with pytest.raises(AlqError, match="ALQ_ERR_NUMERIC"):
        _banded(eng, bad, [0, 64, 128, n], n)
    want = _chain(eng, vec, n)
    got = _banded(eng, vec, [0, 64, 128, n], n)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


def test_argument_errors_are_invalid(eng):
    from active_learning_b200._lib import AlqError
    n = 100
    vec = eng.pdist(torch.rand((n, 5), device="cuda"), condensed=True)
    xy = torch.empty((n, 2), dtype=torch.int32, device="cuda")
    md = torch.empty(n, dtype=torch.float64, device="cuda")
    lib, h, s = eng.lib, eng._h, eng._stream()
    P = ctypes.c_void_p

    def call(cuts, ptrs, nb=None, nn=n, ctx=h, out=True):
        c = np.asarray(cuts, dtype=np.int64)
        arr = (P * max(len(ptrs), 1))(*[P(p) for p in ptrs])
        return lib.alq_ward_nn_chain_banded(ctx, P(c.ctypes.data), arr, len(ptrs) if nb is None else nb, nn,
                                            P(xy.data_ptr() if out else 0), P(md.data_ptr()), s)

    v = vec.data_ptr()
    invalid = 1
    assert call([0, n], [v], ctx=None) == invalid
    assert call([0, n], [v], out=False) == invalid
    assert call([0, 50, 40, n], [v, v, v]) == invalid                  # decreasing cuts
    assert call([1, n], [v]) == invalid                                # not starting at 0
    assert call([0, n - 1], [v]) == invalid                            # not ending at n
    assert call([0, 50, n], [v, 0]) == invalid                         # a band with pairs and no pointer
    assert call([0] + [n] * 9, [v] * 9) == invalid                     # 9 bands
    assert call([0, n], [v], nb=0) == invalid
    assert call([0, n], [v], nn=1) == invalid
    with pytest.raises(AlqError):
        eng.nn_chain_banded([0, 50, n], [vec], n)                       # one band for two
    with pytest.raises(AlqError):
        eng.nn_chain_banded([0, n], [vec[:10]], n)                      # too short
    assert lib.alq_band_alloc(h, 0, ctypes.byref(P()), (ctypes.c_char * 64)()) == invalid
    assert lib.alq_band_free(h, P(0)) == invalid and lib.alq_band_close(h, P(0)) == invalid
    torch.cuda.synchronize()
    # valid edge cases: row n - 1 alone without a pointer, empty bands, eight bands
    want = _chain(eng, vec, n)
    for plan in ([0, n - 1, n], [0, 0, 0, 30, n, n], [0, 1, 2, 3, 4, 5, 6, 64, n]):
        got = _banded(eng, vec, plan, n)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), plan


def _distributed(group, monkeypatch):
    """ShardGroup.ward_labels with layout="distributed" for every call (the sampler's included)."""
    from active_learning_b200 import sharding
    real = sharding.ShardGroup.ward_labels
    chains = []

    def ward_labels(self, x, n_clusters, engine, rows_digest="", layout=None):
        chains.append(x.shape[0])
        return real(self, x, n_clusters, engine, rows_digest, "distributed")

    monkeypatch.setattr(sharding.ShardGroup, "ward_labels", ward_labels)
    return chains


def test_group_of_one_rank_distributed_returns_the_goldens(eng, group, gold, monkeypatch):
    from test_gpu_margin_clustering_sharded import _sampler
    calls = _distributed(group, monkeypatch)
    real_chain = eng.nn_chain
    monkeypatch.setattr(eng, "nn_chain", lambda *a, **k: pytest.fail("the distributed placement gathers no D"))
    for tag in TAGS:
        for h in range(int(gold[f"{tag}_hac_calls"])):
            x = torch.from_numpy(gold[f"{tag}_hac{h}_x"]).cuda()
            assert np.array_equal(group.ward_labels(x, 20, eng, rows_digest="golden"), gold[f"{tag}_hac{h}_labels"])
        s = _sampler(gold, tag, eng)
        for r in range(2):
            np.random.seed(100 + r)
            idx, cost = s._query_sharded(float(gold[f"{tag}_budget"]), group)
            assert [int(i) for i in idx] == gold[f"{tag}_r{r}_picks"].tolist(), (tag, r)
            assert cost == int(gold[f"{tag}_r{r}_cost"])
            s.update(idx, cost)
    assert len(calls) > 5
    monkeypatch.setattr(eng, "nn_chain", real_chain)
    x = torch.from_numpy(_rows(3000, 64, 3)).cuda()
    assert np.array_equal(group.ward_labels(x, 20, eng), eng.ward_labels(x, 20))


def _ipc_worker(rank, world, port, out_path):
    """Both processes on device 0: process 1's band is opened by process 0 through CUDA IPC."""
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    res = {"rank": rank}
    try:
        from active_learning_b200.engine import Engine
        torch.cuda.set_device(0)
        eng = Engine(0)
        torch.empty(1, device="cuda")
        ok = None
    except Exception as exc:                              # noqa: BLE001 -- e.g. an exclusive-process compute mode
        eng, ok = None, f"{type(exc).__name__}: {exc}"
    oks = [None] * world
    dist.all_gather_object(oks, ok)
    if any(oks):
        res["skip"] = "; ".join(o for o in oks if o)
    else:
        from active_learning_b200 import sharding
        group = sharding.ShardGroup()
        gold = dict(np.load(os.path.join(HERE, "golden", "reference_golden_margin_clustering.npz")))
        opened = []
        real_open = eng.band_open

        def band_open(handle, nbytes):
            opened.append(nbytes)
            return real_open(handle, nbytes)

        eng.band_open = band_open
        for tag in TAGS:
            for h in range(int(gold[f"{tag}_hac_calls"])):
                x = torch.from_numpy(gold[f"{tag}_hac{h}_x"]).cuda()
                res[(tag, h)] = group.ward_labels(x, 20, eng, rows_digest="golden", layout="distributed").tolist()
        x = torch.from_numpy(_rows(3000, 64, 3)).cuda()
        res["labels"] = group.ward_labels(x, 20, eng, layout="distributed").tolist()
        res["one_gpu"] = eng.ward_labels(x, 20).tolist()
        res["opened"] = opened
        eng.close()
    all_res = [None] * world
    dist.all_gather_object(all_res, res)
    if rank == 0:
        np.save(out_path, np.array(all_res, dtype=object), allow_pickle=True)
    dist.barrier()
    dist.destroy_process_group()


def _spawn(worker, world):
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    out = os.path.join(tempfile.mkdtemp(), "res.npy")
    mp.spawn(worker, args=(world, port, out), nprocs=world, join=True)
    return list(np.load(out, allow_pickle=True))


def test_two_processes_on_one_gpu_share_a_band_through_cuda_ipc(gold):
    from active_learning_b200.sharding import ward_band_bytes
    results = _spawn(_ipc_worker, 2)
    if "skip" in results[0]:
        pytest.skip(f"this device does not take a second process's context: {results[0]['skip']}")
    for res in results:
        for tag in TAGS:
            for h in range(int(gold[f"{tag}_hac_calls"])):
                assert res[(tag, h)] == gold[f"{tag}_hac{h}_labels"].tolist(), (res["rank"], tag, h)
        assert res["labels"] == res["one_gpu"] == results[0]["one_gpu"]
    assert results[0]["opened"][-1] == ward_band_bytes(3000, 2)[1]      # rank 0 mapped rank 1's band
    assert len(results[0]["opened"]) == 6 and results[1]["opened"] == []


def _nccl_worker(rank, world, port, out_path):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    import torch.distributed as dist
    dist.init_process_group("nccl", rank=rank, world_size=world)
    from active_learning_b200 import sharding
    from active_learning_b200.engine import Engine
    eng = Engine(rank)
    group = sharding.ShardGroup()
    gold = dict(np.load(os.path.join(HERE, "golden", "reference_golden_margin_clustering.npz")))
    res = {}
    for tag in TAGS:
        for h in range(int(gold[f"{tag}_hac_calls"])):
            x = torch.from_numpy(gold[f"{tag}_hac{h}_x"]).cuda()
            res[(tag, h)] = group.ward_labels(x, 20, eng, rows_digest="golden", layout="distributed").tolist()
    # rank 0 reports just its own band's memory: it holds neither layout, the placement rule goes distributed
    n = 3000
    x = torch.from_numpy(_rows(n, 64, 5)).cuda()
    if rank == 0:
        eng._ward_free_bytes = lambda: sharding.ward_band_bytes(n, world)[0] + Engine.WARD_HEADROOM_BYTES
    chains = []
    real_chain = eng.nn_chain_banded
    eng.nn_chain_banded = lambda *a, **k: (chains.append(1), real_chain(*a, **k))[1]
    res["rule"] = group.ward_labels(x, 20, eng).tolist()
    res["chains"] = len(chains)
    all_res = [None] * world
    dist.all_gather_object(all_res, res)
    if rank == 0:
        np.save(out_path, np.array(all_res, dtype=object), allow_pickle=True)
    dist.barrier()
    eng.close()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_distributed_returns_the_goldens_on_every_rank(gold):
    world = min(torch.cuda.device_count(), 8)
    results = _spawn(_nccl_worker, world)
    want = W.ward_labels(_rows(3000, 64, 5)).tolist()
    for r, res in enumerate(results):
        for tag in TAGS:
            for h in range(int(gold[f"{tag}_hac_calls"])):
                assert res[(tag, h)] == gold[f"{tag}_hac{h}_labels"].tolist()
        assert res["rule"] == want
        assert res["chains"] == (1 if r == 0 else 0)
