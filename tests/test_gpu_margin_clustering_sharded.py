"""K7 over bands of rows (alq_pdist_f64_condensed_rows) and their expansion into the square matrix (alq_pdist_f64_expand)
on the H100, and MarginClusteringSampler's sharded path in a group of one rank.

Bands of any plan -- ward_bands(n, G) for G = 1..8, single-row bands, empty bands, cuts off the 64-row tiles -- must
concatenate to alq_pdist_f64_condensed's vector and expand to alq_pdist_f64's matrix bit for bit, and write nothing
outside their range.  A group of one rank (gloo world 1) runs ShardGroup.ward_labels and _query_sharded end to end on
this GPU.  Two or more GPUs: the sampler in an NCCL group (skipped below two GPUs)."""
import ctypes
import os
import socket
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp
from scipy.spatial.distance import pdist as scipy_pdist
from scipy.spatial.distance import squareform

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
TAGS = ("f", "s", "t", "b")


@pytest.fixture(scope="module")
def eng(tmp_path_factory):
    from helpers import one_rank_engine
    with one_rank_engine(tmp_path_factory.mktemp("ward_one_rank")) as e:
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


def _bits(t):
    return t.contiguous().view(torch.int64)


def _splits(n):
    """Band plans over [0, n): ward_bands for 1..8 ranks, then hand-picked ones."""
    from active_learning_b200.sharding import ward_bands
    plans = [ward_bands(n, g) for g in range(1, 9)]
    if n <= 129:
        plans.append(list(range(n + 1)))                                   # every row its own band
    else:
        plans.append([0, 1, 2, 65, 66, n - 1, n])                          # single-row bands at both ends
    plans.append([0, min(5, n), n, n])                                     # an empty band at the end
    plans.append([0, 0, min(5, n), min(5, n), n, n])                       # empty bands between
    plans.append(sorted({0, n} | {c for c in (37, 100, 1000) if c < n}))    # cuts that are not multiples of 64
    return plans


def _x(n, d):
    """(x on the device, x for scipy): d == 'pad' is 17 columns with 3 zero pad columns."""
    if d == "pad":
        x = _rows(n, 17, n + 17)
        return torch.from_numpy(np.pad(x, ((0, 0), (0, 3)))).cuda(), x
    x = _rows(n, d, n * 31 + d)
    return torch.from_numpy(x).cuda(), x


@pytest.mark.parametrize("n", [2, 3, 63, 64, 65, 129, 4097])
@pytest.mark.parametrize("d", [1, 3, 17, "pad"])
def test_bands_of_any_plan_rebuild_the_full_k7_output(eng, n, d):
    from active_learning_b200.sharding import band_pairs
    x, xh = _x(n, d)
    full_c = eng.pdist(x, condensed=True)
    full_s = eng.pdist(x)
    if n <= 129:
        want = scipy_pdist(xh.astype(np.float64))
        assert np.array_equal(full_c.cpu().numpy(), want)
        assert np.array_equal(full_s.cpu().numpy(), squareform(want))
    for plan in _splits(n):
        cat = torch.cat([eng.pdist_rows(x, lo, hi) for lo, hi in zip(plan, plan[1:])])
        assert torch.equal(_bits(cat), _bits(full_c)), plan
        sq = torch.full((n, n), float("nan"), dtype=torch.float64, device="cuda")
        for lo, hi in zip(plan, plan[1:]):
            m = band_pairs(n, lo, hi)
            at = band_pairs(n, 0, lo)
            eng.pdist_expand(full_c[at:at + m], n, lo, hi, sq)
        assert torch.equal(_bits(sq), _bits(full_s)), plan                  # the diagonal included


@pytest.mark.parametrize("n,lo,hi", [(130, 0, 64), (130, 37, 101), (130, 129, 130), (130, 64, 64), (4097, 1000, 1100),
                                     (4097, 4000, 4097)])
def test_band_and_expand_write_nothing_outside_their_range(eng, n, lo, hi):
    from active_learning_b200.sharding import band_pairs
    x = torch.from_numpy(_rows(n, 9, n + lo)).cuda()
    full_c = eng.pdist(x, condensed=True)
    full_s = eng.pdist(x)
    m, at = band_pairs(n, lo, hi), band_pairs(n, 0, lo)
    nan = float("nan")
    out = torch.full((m + 4096,), nan, dtype=torch.float64, device="cuda")
    assert eng.pdist_rows(x, lo, hi, out=out) is out
    assert torch.equal(_bits(out[:m]), _bits(full_c[at:at + m]))
    assert bool(torch.isnan(out[m:]).all())
    # the square matrix, with a leading dimension past n: only rows [lo, hi) of the upper triangle, their mirror and
    # their diagonal are written
    big = torch.full((n, n + 37), nan, dtype=torch.float64, device="cuda")
    eng.pdist_expand(full_c[at:at + m], n, lo, hi, big[:, :n])
    i = torch.arange(n, device="cuda")
    band = (i >= lo) & (i < hi)
    upper = band[:, None] & (i[None, :] >= i[:, None])
    written = upper | upper.T
    sq = big[:, :n]
    assert torch.equal(_bits(sq[written]), _bits(full_s[written]))
    assert bool(torch.isnan(sq[~written]).all()) and bool(torch.isnan(big[:, n:]).all())


def test_three_bands_past_2_31_entries_at_70000_rows(eng):
    """n (n - 1) / 2 = 2.45e9 > 2^31: the bands of ward_bands(n, 3), each into its slice of one vector, are
    alq_pdist_f64_condensed's vector bit for bit (two 19.6 GB vectors)."""
    from active_learning_b200.sharding import band_pairs, ward_bands
    n = 70000
    if eng._ward_free_bytes() < 2 * 4 * n * (n - 1) + (2 << 30):
        pytest.skip(f"needs {2 * 4 * n * (n - 1)} bytes of free device memory")
    x = torch.from_numpy(_rows(n, 16, n)).cuda()
    full = eng.pdist(x, condensed=True)
    cat = torch.full_like(full, float("nan"))
    b = ward_bands(n, 3)
    assert b[1] > 0 and band_pairs(n, 0, b[2]) < 1 << 31 < full.shape[0]     # the last band crosses 2^31
    for lo, hi in zip(b, b[1:]):
        at = band_pairs(n, 0, lo)
        eng.pdist_rows(x, lo, hi, out=cat[at:at + band_pairs(n, lo, hi)])
    assert torch.equal(_bits(cat), _bits(full))
    del cat, full
    torch.cuda.empty_cache()


def test_three_bands_expand_to_the_square_matrix_at_47000_rows(eng):
    """n^2 = 2.2e9 > 2^31 entries of the square matrix (17.7 GB, twice) from the three bands of ward_bands(n, 3)."""
    from active_learning_b200.sharding import band_pairs, ward_bands
    n = 47000
    b = ward_bands(n, 3)
    need = 2 * 8 * n * n + 8 * max(band_pairs(n, lo, hi) for lo, hi in zip(b, b[1:]))
    if eng._ward_free_bytes() < need + (1 << 30):
        pytest.skip(f"needs {need} bytes of free device memory")
    x = torch.from_numpy(_rows(n, 16, n)).cuda()
    full = eng.pdist(x)
    sq = torch.full_like(full, float("nan"))
    for lo, hi in zip(b, b[1:]):
        band = eng.pdist_rows(x, lo, hi)
        assert band.shape[0] == band_pairs(n, lo, hi)
        eng.pdist_expand(band, n, lo, hi, sq)
        del band
    assert torch.equal(_bits(sq), _bits(full))
    del sq, full
    torch.cuda.empty_cache()


def test_argument_errors_are_invalid(eng):
    from active_learning_b200._lib import AlqError
    n, d = 100, 5
    x = torch.rand((n, d), device="cuda")
    out = torch.empty(n * n, dtype=torch.float64, device="cuda")
    sq = torch.empty((n, n), dtype=torch.float64, device="cuda")
    lib, h, null, s = eng.lib, eng._h, ctypes.c_void_p(0), eng._stream()
    xp, op, sp = ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(sq.data_ptr())
    invalid = 1
    rows = lib.alq_pdist_f64_condensed_rows
    assert rows(None, xp, n, d, d, 0, n, op, s) == invalid
    assert rows(h, null, n, d, d, 0, n, op, s) == invalid
    assert rows(h, xp, n, d, d, 0, n, null, s) == invalid
    assert rows(h, xp, n, d, d, -1, n, op, s) == invalid
    assert rows(h, xp, n, d, d, 0, n + 1, op, s) == invalid
    assert rows(h, xp, n, d, d, 7, 6, op, s) == invalid
    assert rows(h, xp, n, d, d - 1, 0, n, op, s) == invalid
    assert rows(h, xp, 65535 * 64 + 1, d, d, 0, 1, op, s) == invalid
    assert rows(h, xp, n, d, d, 7, 7, op, s) == 0                          # an empty band is valid
    expand = lib.alq_pdist_f64_expand
    assert expand(None, op, n, 0, n, sp, n, s) == invalid
    assert expand(h, null, n, 0, n, sp, n, s) == invalid
    assert expand(h, op, n, 0, n, null, n, s) == invalid
    assert expand(h, op, n, -1, n, sp, n, s) == invalid
    assert expand(h, op, n, 0, n + 1, sp, n, s) == invalid
    assert expand(h, op, n, 7, 6, sp, n, s) == invalid
    assert expand(h, op, n, 0, n, sp, n - 1, s) == invalid
    assert expand(h, op, n, 7, 7, sp, n, s) == 0
    for lo, hi in ((-1, 5), (0, n + 1), (6, 5)):
        with pytest.raises(AlqError):
            eng.pdist_rows(x, lo, hi)
        with pytest.raises(AlqError):
            eng.pdist_expand(out, n, lo, hi, sq)
    with pytest.raises(AlqError):
        eng.pdist_rows(x, 0, n, out=torch.empty(10, dtype=torch.float64, device="cuda"))
    with pytest.raises(AlqError):
        eng.pdist_expand(out[:10], n, 0, n, sq)
    with pytest.raises(AlqError):
        eng.pdist_expand(out, n, 0, n, sq[:, :n - 1])
    torch.cuda.synchronize()
    x2 = torch.from_numpy(_rows(40, 3, 40)).cuda()                        # the context is still usable
    assert np.array_equal(eng.pdist_rows(x2, 0, 40).cpu().numpy(), scipy_pdist(x2.cpu().numpy().astype(np.float64)))


def _condensed_only(eng, monkeypatch, layouts):
    """The free-bytes probe reports just enough for the condensed vector of each call (it needs no staging on rank 0)."""
    from active_learning_b200 import sharding
    real_labels, real_chain = sharding.ShardGroup.ward_labels, eng.nn_chain

    def ward_labels(self, x, n_clusters, engine, rows_digest=""):
        n = x.shape[0]
        monkeypatch.setattr(engine, "_ward_free_bytes", lambda: engine.ward_condensed_bytes(n))
        return real_labels(self, x, n_clusters, engine, rows_digest)

    def nn_chain(dist, n=None):
        layouts.append(dist.dim())
        return real_chain(dist, n)

    monkeypatch.setattr(sharding.ShardGroup, "ward_labels", ward_labels)
    monkeypatch.setattr(eng, "nn_chain", nn_chain)


@pytest.mark.parametrize("layout", ["square", "condensed"])
def test_group_ward_labels_equal_the_engine_and_sklearns_goldens(eng, group, gold, monkeypatch, layout):
    from active_learning_b200 import sharding
    layouts = []
    if layout == "condensed":
        _condensed_only(eng, monkeypatch, layouts)
    else:
        real = eng.nn_chain
        monkeypatch.setattr(eng, "nn_chain", lambda dist, n=None: (layouts.append(dist.dim()), real(dist, n))[1])
    monkeypatch.setattr(sharding, "WARD_CHUNK_BYTES", 8 * 5000)          # several chunks through the two buffers
    for tag in TAGS:
        for h in range(int(gold[f"{tag}_hac_calls"])):
            x = torch.from_numpy(gold[f"{tag}_hac{h}_x"]).cuda()
            got = group.ward_labels(x, 20, eng, rows_digest="golden")
            assert np.array_equal(got, gold[f"{tag}_hac{h}_labels"]), (tag, h)
    assert layouts == [2 if layout == "square" else 1] * len(layouts) and len(layouts) == 5
    monkeypatch.undo()
    x = torch.from_numpy(_rows(3000, 64, 3)).cuda()                       # a larger pool against the one-GPU call
    assert np.array_equal(group.ward_labels(x, 20, eng), eng.ward_labels(x, 20))


def _sampler(gold, tag, eng):
    from helpers import HeadNet, make_strategy
    emb = torch.from_numpy(gold[f"{tag}_emb"])
    kw = {}
    if int(gold[f"{tag}_subset"]) >= 0:
        kw["subset_unlabeled"] = int(gold[f"{tag}_subset"])
    if f"{tag}_logits" in gold:
        logits, net = torch.from_numpy(gold[f"{tag}_logits"]), None
    else:
        logits, net = None, HeadNet(emb, torch.from_numpy(gold[f"{tag}_weight"]), torch.from_numpy(gold[f"{tag}_bias"]))
    return make_strategy("MarginClusteringSampler", logits, emb, gold[f"{tag}_eval"], gold[f"{tag}_labeled"],
                         int(gold[f"{tag}_bs"]), engine=eng, net=net, **kw)


@pytest.mark.parametrize("tag", TAGS)
def test_query_sharded_in_a_group_of_one_rank_replays_the_goldens(eng, group, gold, tag):
    s = _sampler(gold, tag, eng)
    for r in range(2):
        np.random.seed(100 + r)
        idx, cost = s._query_sharded(float(gold[f"{tag}_budget"]), group)
        assert [int(i) for i in idx] == gold[f"{tag}_r{r}_picks"].tolist(), (tag, r)
        assert cost == int(gold[f"{tag}_r{r}_cost"])
        s.update(idx, cost)


def _worker(rank, world, port, out_path):
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
        s = _sampler(gold, tag, eng)
        s._shard_group = group
        for r in range(2):
            np.random.seed(100 + r)
            idx, cost = s.query(float(gold[f"{tag}_budget"]))
            res[(tag, r)] = ([int(i) for i in idx], int(cost))
            s.update(idx, cost)
    sharding.WARD_CHUNK_BYTES = 8 * 5000
    x = torch.from_numpy(_rows(3000, 64, 3)).cuda()
    res["labels"] = group.ward_labels(x, 20, eng).tolist()
    res["one_gpu"] = eng.ward_labels(x, 20).tolist()
    all_res = [None] * world
    dist.all_gather_object(all_res, res)
    if rank == 0:
        np.save(out_path, np.array(all_res, dtype=object), allow_pickle=True)
    dist.barrier()
    eng.close()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_sampler_returns_the_goldens_on_every_rank(gold):
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    out = os.path.join(tempfile.mkdtemp(), "res.npy")
    world = min(torch.cuda.device_count(), 4)
    mp.spawn(_worker, args=(world, port, out), nprocs=world, join=True)
    results = list(np.load(out, allow_pickle=True))
    for res in results:
        for tag in TAGS:
            for r in range(2):
                assert res[(tag, r)] == (gold[f"{tag}_r{r}_picks"].tolist(), int(gold[f"{tag}_r{r}_cost"]))
        assert res["labels"] == res["one_gpu"] == results[0]["one_gpu"]
