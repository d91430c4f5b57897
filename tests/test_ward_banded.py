"""MarginClusteringSampler's distributed Ward placement on the CPU: the placement rule (ward_group_placement), the NumPy
twin of K8's banded addressing against the oracle and scipy, and ShardGroup.ward_labels's distributed orchestration in
gloo groups of 2 and 3 ranks.  There the engine is a twin whose band memory is an np.memmap file under a shared temporary
directory and whose "IPC handle" is that file's path, so rank 0's K8 (the banded twin) reads the peers' bands in place."""
import os
import socket
import sys
import tempfile
import uuid

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import ward_oracle as W
from ward_banded_twin import split_condensed, ward_nn_chain_banded

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
TAGS = ("f", "s", "t", "b")
EVENTS = []                # this process's record: band allocations, K7, handle exchange, K8, broadcasts, frees


def load_gold():
    return dict(np.load(os.path.join(HERE, "golden", "reference_golden_margin_clustering.npz")))


# ---- placement ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1000, 80000, 115846, 200000, 390000])
def test_placement_table(n):
    from active_learning_b200._lib import AlqError
    from active_learning_b200.engine import Engine
    from active_learning_b200.sharding import ward_band_bytes, ward_group_placement
    H, staging = Engine.WARD_HEADROOM_BYTES, 4 << 30
    sq, cond = Engine.ward_bytes(n), Engine.ward_condensed_bytes(n)
    for world in range(1, 9):
        band = [b + H for b in ward_band_bytes(n, world)]
        assert sum(ward_band_bytes(n, world)) == 4 * n * (n - 1)
        big = [1 << 62] * (world - 1)
        assert ward_group_placement(n, [sq + staging] + big, staging) == "square"
        assert ward_group_placement(n, [sq + staging - 1] + big, staging) == "condensed"
        assert ward_group_placement(n, [cond] + big, staging) == "condensed"
        # rank 0 one byte short of the vector: distributed when every rank holds its own band plus the headroom
        exact = [min(b, cond - 1) if r == 0 else b for r, b in enumerate(band)]
        if world == 1 or band[0] > cond - 1:
            with pytest.raises(AlqError):
                ward_group_placement(n, exact, staging)
            continue
        assert ward_group_placement(n, exact, staging) == "distributed"
        assert ward_group_placement(n, [cond - 1] + big, staging) == "distributed"    # uneven: plenty on peers
        for r in range(world):                                             # any rank one byte short: nothing fits
            short = list(exact)
            short[r] -= 1
            with pytest.raises(AlqError) as e:
                ward_group_placement(n, short, staging)
            msg = str(e.value)
            assert f"n={n}" in msg and str(sq) in msg and str(cond) in msg and str(max(band)) in msg
        with pytest.raises(AlqError, match=str(cond)):                     # an engine without the band calls
            ward_group_placement(n, exact, staging, distributed=False)


def test_placement_rank0_fitting_a_layout_wins_over_distributed():
    from active_learning_b200.engine import Engine
    from active_learning_b200.sharding import ward_group_placement
    n = 2000
    cond = Engine.ward_condensed_bytes(n)
    assert ward_group_placement(n, [cond, 0, 0], 0) == "condensed"        # peers with no memory at all: unchanged
    assert ward_group_placement(n, [1 << 62, 0], 1 << 40) == "square"


def test_eight_h100s_hold_about_390000_rows_distributed():
    """Computed from memory, not run: 80 GB per card (80e9 bytes free) and 1 GiB headroom per rank."""
    from active_learning_b200._lib import AlqError
    from active_learning_b200.sharding import ward_group_placement
    free = [80 * 10 ** 9] * 8
    assert ward_group_placement(390000, free, 0) == "distributed"
    assert ward_group_placement(140000, free[:1], 0) == "condensed"       # one card's limit
    with pytest.raises(AlqError):
        ward_group_placement(145000, free[:1], 0)
    with pytest.raises(AlqError):
        ward_group_placement(420000, free, 0)


# ---- the banded addressing ------------------------------------------------------------------------------------------
def _rows(n, d, seed):
    rng = np.random.default_rng(seed)
    return np.maximum(rng.standard_normal((n, d)), 0).astype(np.float32)


@pytest.mark.parametrize("n", [2, 3, 63, 64, 65, 129, 300])
def test_banded_twin_equals_the_oracle_and_scipy(n):
    hierarchy = pytest.importorskip("scipy.cluster.hierarchy")
    from scipy.spatial.distance import pdist
    from test_gpu_margin_clustering_sharded import _splits
    x = _rows(n, 5, n)
    vec = pdist(x.astype(np.float64))
    want_xy, want_md, _ = W.ward_nn_chain(W.pdist_square(x))
    Z = hierarchy.ward(x)
    plans = [p for p in _splits(n) if len(p) - 1 <= 8]
    assert len(plans) >= 10
    for plan in plans:
        bands = split_condensed(vec, plan, n)
        xy, md = ward_nn_chain_banded(plan, bands, n)
        assert np.array_equal(xy, want_xy) and np.array_equal(md, want_md), plan
        assert np.array_equal(W.linkage_from_merges(xy, md, n), Z), plan


# ---- the distributed orchestration in a gloo group ------------------------------------------------------------------
class MemmapBand:
    """Engine.WardBand's twin: a float64 np.memmap file; its "IPC handle" is the file's path."""

    def __init__(self, path, nbytes, owned):
        self.path, self.nbytes, self.owned, self.handle = path, int(nbytes), owned, path.encode()
        self.arr = np.memmap(path, dtype=np.float64, mode="r+", shape=(self.nbytes // 8,))

    def tensor(self):
        return torch.from_numpy(self.arr)

    def release(self):
        if self.arr is None:
            return
        self.arr.flush()
        self.arr = None
        EVENTS.append(("free" if self.owned else "close", self.path))
        if self.owned:
            os.remove(self.path)


def make_engine(tmp):
    from test_margin_clustering import WardOracleEngine
    from test_margin_clustering_sharded import band_twin

    class BandedTwinEngine(WardOracleEngine):
        """WardOracleEngine with Engine's band (pdist_rows), band-memory and banded chain calls as twins."""

        def __init__(self):
            self.free = 1 << 50
            self.fail_alloc = self.fail_chain = False

        def _ward_free_bytes(self):
            return self.free

        def pdist_rows(self, x, row_lo, row_hi, out=None):
            v = torch.from_numpy(band_twin(x.numpy(), int(row_lo), int(row_hi)))
            if int(row_hi) > int(row_lo):
                EVENTS.append(("k7", int(row_lo), int(row_hi)))
            if out is None:
                return v
            out[:len(v)] = v
            return out

        def band_alloc(self, nbytes):
            from active_learning_b200._lib import AlqError
            if self.fail_alloc:
                raise AlqError("alq_band_alloc: ALQ_ERR_NOMEM: allocation failed (test)")
            path = os.path.join(tmp, f"band-{uuid.uuid4().hex}")
            with open(path, "wb") as f:
                f.truncate(int(nbytes))
            EVENTS.append(("alloc", path))
            return MemmapBand(path, nbytes, owned=True)

        def band_open(self, handle, nbytes):
            EVENTS.append(("open", handle.decode()))
            return MemmapBand(handle.decode(), nbytes, owned=False)

        def nn_chain_banded(self, row_cuts, bands, n):
            from active_learning_b200._lib import AlqError
            EVENTS.append(("k8", [None if b is None else b.path for b in bands]))
            if self.fail_chain:
                raise AlqError("alq_ward_nn_chain_banded: ALQ_ERR_NUMERIC: no finite distance (test)")
            xy, md = ward_nn_chain_banded(row_cuts, [None if b is None else b.arr for b in bands], n)
            return torch.from_numpy(xy.astype(np.int32)), torch.from_numpy(md)

        def nn_chain(self, dist, n=None):
            raise AssertionError("the distributed placement never gathers the distances")

    return BandedTwinEngine()


def _worker(rank, world, port, tmp, out_path):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from active_learning_b200 import sharding
    from active_learning_b200._lib import AlqError
    from active_learning_b200.engine import Engine
    from test_margin_clustering_sharded import sampler
    gold = load_gold()
    group = sharding.ShardGroup()
    res = {"rank": rank}
    sent = []
    real = {k: getattr(dist, k) for k in ("isend", "irecv", "send", "recv", "broadcast_object_list")}
    for k in ("isend", "irecv", "send", "recv"):
        setattr(dist, k, lambda *a, _k=k, **kw: (sent.append(_k), real[_k](*a, **kw))[1])

    def broadcast(*a, **kw):
        EVENTS.append(("broadcast",))
        return real["broadcast_object_list"](*a, **kw)

    dist.broadcast_object_list = broadcast
    real_labels = group.ward_labels

    def tight(x, n_clusters, engine, rows_digest="", layout=None):
        """Every rank's free memory holds its band plus the headroom, rank 0 fits neither of its layouts: the
        placement rule picks the distributed one by itself."""
        engine.free = max(sharding.ward_band_bytes(x.shape[0], world)) + Engine.WARD_HEADROOM_BYTES
        return real_labels(x, n_clusters, engine, rows_digest, layout)

    # the sampler's two golden rounds, placed by the rule
    group.ward_labels = tight
    for tag in TAGS:
        s = sampler(gold, tag, make_engine(tmp), group)
        for r in range(2):
            np.random.seed(100 + r)
            EVENTS.clear()
            idx, cost = s.query(float(gold[f"{tag}_budget"]))
            res[(tag, r)] = ([int(i) for i in idx], int(cost), list(EVENTS))
            s.update(idx, cost)
    del group.ward_labels
    # the group call on every golden HAC input, forced and by the rule
    for how in ("forced", "rule"):
        for tag in TAGS:
            for h in range(int(gold[f"{tag}_hac_calls"])):
                x = torch.from_numpy(gold[f"{tag}_hac{h}_x"])
                EVENTS.clear()
                if how == "forced":
                    labels = group.ward_labels(x, 20, make_engine(tmp), rows_digest="golden", layout="distributed")
                else:
                    labels = tight(x, 20, make_engine(tmp), rows_digest="golden")
                res[(how, tag, h)] = (labels, list(EVENTS))
    # a peer cannot reserve its band: every rank raises before any band is computed, forced and by the rule
    for how in ("forced", "rule"):
        eng = make_engine(tmp)
        eng.fail_alloc = rank == world - 1
        EVENTS.clear()
        try:
            x = torch.from_numpy(gold["f_hac0_x"])
            if how == "forced":
                group.ward_labels(x, 20, eng, rows_digest="golden", layout="distributed")
            else:
                tight(x, 20, eng, rows_digest="golden")
            res[("alloc_failure", how)] = ("no error", [])
        except AlqError as exc:
            res[("alloc_failure", how)] = (str(exc), list(EVENTS))
    # K8 fails on rank 0: every rank raises rank 0's message, and every band is still freed
    eng = make_engine(tmp)
    eng.fail_chain = True
    EVENTS.clear()
    try:
        group.ward_labels(torch.from_numpy(gold["b_hac0_x"]), 20, eng, rows_digest="golden", layout="distributed")
        res["chain_failure"] = ("no error", [])
    except AlqError as exc:
        res["chain_failure"] = (str(exc), list(EVENTS))
    # ranks that disagree on the placement they ask for
    try:
        group.ward_labels(torch.from_numpy(gold["b_hac0_x"]), 20, make_engine(tmp), rows_digest="golden",
                          layout="distributed" if rank == 0 else None)
        res["layout_mismatch"] = "no error"
    except AlqError as exc:
        res["layout_mismatch"] = str(exc)
    for k, v in real.items():
        setattr(dist, k, v)
    res["sent"] = sent
    all_res = [None] * world
    dist.all_gather_object(all_res, res)
    if rank == 0:
        np.save(out_path, np.array(all_res, dtype=object), allow_pickle=True)
    dist.barrier()
    dist.destroy_process_group()


@pytest.fixture(scope="module")
def gold():
    return load_gold()


@pytest.fixture(scope="module")
def lib_built():
    from active_learning_b200 import _lib, build
    if not os.path.exists(_lib.LIB_PATH):                 # alq_ward_labels is host-only: no GPU needed
        build.build()


@pytest.fixture(scope="module", params=[2, 3])
def group_results(request, lib_built, tmp_path_factory):
    world = request.param
    tmp = str(tmp_path_factory.mktemp(f"bands{world}"))
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    out = os.path.join(tempfile.mkdtemp(), "res.npy")
    mp.spawn(_worker, args=(world, port, tmp, out), nprocs=world, join=True)
    return world, list(np.load(out, allow_pickle=True)), tmp


def _check_lifetime(events, rank, world, n):
    """One band per rank with pairs, K7 once into it, K8 on rank 0 over every band, no peer free before the broadcast."""
    from active_learning_b200.sharding import band_pairs, ward_bands
    b = ward_bands(n, world)
    kinds = [e[0] for e in events]
    has = band_pairs(n, b[rank], b[rank + 1]) > 0
    assert kinds.count("alloc") == kinds.count("free") == int(has)
    assert [e for e in events if e[0] == "k7"] == ([("k7", b[rank], b[rank + 1])] if has else [])
    if has:
        assert kinds.index("alloc") < kinds.index("k7") < kinds.index("broadcast") < kinds.index("free")
    if rank == 0:
        (k8,) = [e for e in events if e[0] == "k8"]
        peers = k8[1][1:]
        assert [p is not None for p in peers] == [band_pairs(n, b[r], b[r + 1]) > 0 for r in range(1, world)]
        opened = [e[1] for e in events if e[0] == "open"]
        assert [p for p in peers if p] == opened
        closes = [i for i, e in enumerate(events) if e[0] == "close"]
        assert sorted(events[i][1] for i in closes) == sorted(opened)
        assert kinds.index("k8") < kinds.index("broadcast") and all(i < kinds.index("broadcast") for i in closes)
    else:
        assert "k8" not in kinds and "open" not in kinds


def test_every_rank_returns_the_golden_picks_with_the_bands_left_in_place(gold, group_results):
    world, results, tmp = group_results
    assert [r["rank"] for r in results] == list(range(world))
    for tag in TAGS:
        for r in range(2):
            clusters = r == 0 or int(gold[f"{tag}_subset"]) >= 0
            for res in results:
                picks, cost, events = res[(tag, r)]
                assert picks == gold[f"{tag}_r{r}_picks"].tolist() and cost == int(gold[f"{tag}_r{r}_cost"])
                if clusters:
                    n = len(gold[f"{tag}_hac{r if r < int(gold[f'{tag}_hac_calls']) else 0}_x"])
                    _check_lifetime(events, res["rank"], world, n)
                else:
                    assert events == []
    assert os.listdir(tmp) == []                                          # every band freed


def test_group_labels_are_the_goldens_forced_and_by_the_rule(gold, group_results):
    world, results, _ = group_results
    for how in ("forced", "rule"):
        for tag in TAGS:
            for h in range(int(gold[f"{tag}_hac_calls"])):
                for res in results:
                    labels, events = res[(how, tag, h)]
                    assert np.array_equal(labels, gold[f"{tag}_hac{h}_labels"]), (how, tag, h)
                    _check_lifetime(events, res["rank"], world, len(gold[f"{tag}_hac{h}_x"]))


def test_no_point_to_point_transfer_is_posted(group_results):
    _, results, _ = group_results
    for res in results:
        assert res["sent"] == []


def test_a_failed_band_reservation_raises_on_every_rank_before_any_band_is_computed(group_results):
    world, results, _ = group_results
    for how in ("forced", "rule"):
        for res in results:
            msg, events = res[("alloc_failure", how)]
            assert "could not reserve" in msg and f"rank {world - 1}" in msg and "ALQ_ERR_NOMEM" in msg, msg
            kinds = [e[0] for e in events]
            assert "k7" not in kinds and "k8" not in kinds
            assert kinds.count("alloc") == kinds.count("free")


def test_a_chain_failure_raises_rank0s_message_everywhere_and_frees_every_band(group_results):
    world, results, tmp = group_results
    for res in results:
        msg, events = res["chain_failure"]
        assert "ward_labels on rank 0" in msg and "ALQ_ERR_NUMERIC" in msg
        kinds = [e[0] for e in events]
        assert kinds.count("alloc") == kinds.count("free")
        if "free" in kinds:
            assert kinds.index("broadcast") < kinds.index("free")
    assert os.listdir(tmp) == []


def test_ranks_asking_for_different_placements_raise_everywhere(group_results):
    _, results, _ = group_results
    for res in results:
        assert "disagree on layout" in res["layout_mismatch"]
