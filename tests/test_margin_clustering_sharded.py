"""MarginClusteringSampler in a ShardGroup of 2 and 3 ranks, on the CPU (gloo): each rank forwards its row_range of the
HAC rows, the margins (and, in a round that clusters, the embeddings) are replicated with all_gather_rows, and
ShardGroup.ward_labels splits K7 by ward_bands, sends the bands to rank 0 in chunks, runs K8 there and broadcasts the
labels.  The engine is the NumPy twin (tests/ward_oracle.py) with the band, expand and chain calls of Engine; every rank
must return the reference's picks, and the distances rank 0 assembles must be scipy's."""
import os
import socket
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import ward_oracle as W

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
TAGS = ("f", "s", "t", "b")
SMALL_CHUNK = 8 * 700              # WARD_CHUNK_BYTES that cuts every band of the goldens into several chunks


def load_gold():
    return dict(np.load(os.path.join(HERE, "golden", "reference_golden_margin_clustering.npz")))


def band_twin(x, lo, hi):
    """Rows [lo, hi) of scipy's condensed vector, with W.pdist_square's arithmetic."""
    x = np.asarray(x, dtype=np.float64)
    parts = []
    for i in range(lo, hi):
        diff = x[i] - x[i + 1:]
        parts.append(np.sqrt(np.cumsum(diff * diff, axis=1)[:, -1]) if len(diff) else np.empty(0))
    return np.concatenate(parts) if parts else np.empty(0)


def make_engine():
    from test_margin_clustering import WardOracleEngine

    class BandTwinEngine(WardOracleEngine):
        """WardOracleEngine with Engine's band (pdist_rows), expand (pdist_expand) and chain (nn_chain) calls as NumPy
        twins; records the non-empty bands computed and the distances handed to the chain."""

        def __init__(self):
            self.free = 1 << 50
            self.bands, self.assembled = [], []
            self.fail_chain = False

        def _ward_free_bytes(self):
            return self.free

        def pdist_rows(self, x, row_lo, row_hi, out=None):
            v = torch.from_numpy(band_twin(x.numpy(), int(row_lo), int(row_hi)))
            if int(row_hi) > int(row_lo):
                self.bands.append((int(row_lo), int(row_hi)))
            if out is None:
                return v
            out[:len(v)] = v
            return out

        def pdist_expand(self, rows, n, row_lo, row_hi, dist):
            r = rows.numpy()
            at = 0
            for i in range(int(row_lo), int(row_hi)):
                m = n - 1 - i
                dist[i, i + 1:n] = torch.from_numpy(r[at:at + m])
                dist[i + 1:n, i] = torch.from_numpy(r[at:at + m])
                dist[i, i] = 0.0
                at += m
            return dist

        def nn_chain(self, dist, n=None):
            from active_learning_b200._lib import AlqError
            from scipy.spatial.distance import squareform
            self.assembled.append(dist.numpy().copy())
            if self.fail_chain:
                raise AlqError("alq_ward_nn_chain failed with ALQ_ERR_NUMERIC (test)")
            D = dist.numpy() if dist.dim() == 2 else squareform(dist.numpy())
            xy, md, _ = W.ward_nn_chain(D[:n, :n])
            return torch.from_numpy(xy.astype(np.int32)), torch.from_numpy(md)

    return BandTwinEngine()


def condensed_only_free(n):
    """Free bytes under which rank 0 fits scipy's condensed vector (which needs no staging) but not the n x n matrix."""
    from active_learning_b200.engine import Engine
    free = Engine.ward_condensed_bytes(n)
    assert free < Engine.ward_bytes(n)
    return free


def sampler(gold, tag, eng, group=None):
    from test_margin_clustering import _sampler
    s = _sampler(gold, tag, eng)
    s._shard_group = group
    s.forwarded = []
    inner = s._forward_pool

    def recording(idxs, *a, **k):
        s.forwarded.append([int(i) for i in idxs])
        return inner(idxs, *a, **k)

    s._forward_pool = recording
    return s


def run_rounds(gold, tag, eng, group=None):
    """The golden's two rounds; per round the picks, the cost, the rows forwarded, the all_gather_rows shapes, the
    bands K7 computed on this rank and the distances K8 got."""
    s = sampler(gold, tag, eng, group)
    gathers = []
    if group is not None:
        inner = group.all_gather_rows

        def gather(t, counts):
            gathers.append(tuple(t.shape[1:]))
            return inner(t, counts)

        group.all_gather_rows = gather
    out = []
    for r in range(2):
        np.random.seed(100 + r)
        s.forwarded, eng.bands, eng.assembled = [], [], []
        gathers.clear()
        idx, cost = s.query(float(gold[f"{tag}_budget"]))
        out.append({"picks": [int(i) for i in idx], "cost": int(cost), "forwarded": s.forwarded,
                    "gathers": list(gathers), "bands": list(eng.bands), "assembled": list(eng.assembled)})
        s.update(idx, cost)
    if group is not None:
        del group.all_gather_rows
    return out


def _worker(rank, world, port, out_path):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from active_learning_b200 import sharding
    from active_learning_b200._lib import AlqError
    gold = load_gold()
    group = sharding.ShardGroup()
    res = {"rank": rank}
    for tag in TAGS:
        res[tag] = run_rounds(gold, tag, make_engine(), group)
    # the group call alone on every golden HAC input, both layouts, the bands cut into several chunks each
    real_chunk, real_irecv = sharding.WARD_CHUNK_BYTES, dist.irecv
    received = []

    def irecv(tensor, src=None, **kw):                    # rank 0's receives, in the order they are posted
        received.append((int(src), int(tensor.numel())))
        return real_irecv(tensor, src=src, **kw)

    dist.irecv = irecv
    for chunk in (real_chunk, SMALL_CHUNK):
        sharding.WARD_CHUNK_BYTES = chunk
        for layout in ("square", "condensed"):
            for tag in TAGS:
                for h in range(int(gold[f"{tag}_hac_calls"])):
                    x = gold[f"{tag}_hac{h}_x"]
                    eng = make_engine()
                    if layout == "condensed":
                        eng.free = condensed_only_free(len(x))
                    received.clear()
                    labels = group.ward_labels(torch.from_numpy(x), 20, eng, rows_digest="golden")
                    res[("labels", chunk, layout, tag, h)] = (labels, eng.bands, eng.assembled, list(received))
    sharding.WARD_CHUNK_BYTES, dist.irecv = real_chunk, real_irecv
    # rows that differ between the ranks (a different subset_unlabeled draw): AlqError everywhere, no band computed
    eng = make_engine()
    s = sampler(gold, "s", eng, group)
    np.random.seed(100 + rank)
    try:
        s.query(float(gold["s_budget"]))
        res["mismatch"] = "no error"
    except AlqError as exc:
        res["mismatch"] = (str(exc), list(eng.bands), len(eng.assembled))
    # K8 fails on rank 0: every rank raises rank 0's error
    eng = make_engine()
    eng.fail_chain = True
    try:
        group.ward_labels(torch.from_numpy(gold["f_hac0_x"]), 20, eng, rows_digest="golden")
        res["chain_failure"] = "no error"
    except AlqError as exc:
        res["chain_failure"] = str(exc)
    # sklearn's ValueErrors, on every rank and before any collective
    errors = []
    bad = gold["f_hac0_x"].copy()
    bad[7, 3] = np.inf
    for x in (bad, gold["f_hac0_x"][:19]):
        try:
            group.ward_labels(torch.from_numpy(x), 20, make_engine())
            errors.append("no error")
        except ValueError as exc:
            errors.append(str(exc))
    res["value_errors"] = errors
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


@pytest.fixture(scope="module")
def single(gold, lib_built):
    """The same rounds in one process without a group."""
    return {tag: run_rounds(gold, tag, make_engine()) for tag in TAGS}


def run_group(world):
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    out = os.path.join(tempfile.mkdtemp(), "res.npy")
    mp.spawn(_worker, args=(world, port, out), nprocs=world, join=True)
    return list(np.load(out, allow_pickle=True))


@pytest.fixture(scope="module", params=[2, 3])
def group_results(request, lib_built):
    return request.param, run_group(request.param)


def test_single_process_rounds_are_the_goldens(gold, single):
    for tag in TAGS:
        for r in range(2):
            assert single[tag][r]["picks"] == gold[f"{tag}_r{r}_picks"].tolist()
            assert single[tag][r]["bands"] == []                          # no group: the one-GPU ward_labels


def test_every_rank_returns_the_goldens_and_forwards_only_its_rows(gold, single, group_results):
    world, results = group_results
    assert [r["rank"] for r in results] == list(range(world))
    for tag in TAGS:
        for r in range(2):
            rows = single[tag][r]["forwarded"][0]                         # the HAC rows of this round
            n = len(rows)
            for res in results:
                got = res[tag][r]
                assert got["picks"] == gold[f"{tag}_r{r}_picks"].tolist(), (tag, r, res["rank"])
                assert got["cost"] == int(gold[f"{tag}_r{r}_cost"])
                q = res["rank"]
                lo, hi = q * (n // world) + min(q, n % world), (q + 1) * (n // world) + min(q + 1, n % world)
                assert got["forwarded"] == [rows[lo:hi]]


def test_only_a_round_that_clusters_gathers_embeddings_and_runs_k7(gold, group_results):
    from active_learning_b200.sharding import ward_bands, ward_chunks
    world, results = group_results
    for tag in TAGS:
        for r in range(2):
            clusters = r == 0 or int(gold[f"{tag}_subset"]) >= 0
            for res in results:
                got = res[tag][r]
                width = gold[f"{tag}_emb"].shape[1]
                want = [()] + ([((width + 3) & ~3,)] if clusters else [])  # the margins, then the padded embeddings
                assert got["gathers"] == want, (tag, r)
                if not clusters:
                    assert got["bands"] == [] and got["assembled"] == []
                else:
                    n = len(gold[f"{tag}_hac{r if r < int(gold[f'{tag}_hac_calls']) else 0}_x"])
                    b = ward_bands(n, world)
                    q = res["rank"]
                    assert got["bands"] == [c for c in ward_chunks(n, b[q], b[q + 1], 1 << 30) if c[1] > c[0]]
                    assert len(got["assembled"]) == (1 if res["rank"] == 0 else 0)      # K8 on rank 0 only


def test_rank0_assembles_scipys_distances_in_both_layouts(gold, group_results):
    from scipy.spatial.distance import pdist
    from active_learning_b200.sharding import band_pairs, ward_bands, ward_chunks, ward_receive_order
    world, results = group_results
    assert len(ward_chunks(328, *ward_bands(328, world)[:2], SMALL_CHUNK)) > 2
    for chunk in sorted({k[1] for k in results[0] if isinstance(k, tuple)}):
        for layout in ("square", "condensed"):
            for tag in TAGS:
                for h in range(int(gold[f"{tag}_hac_calls"])):
                    x = gold[f"{tag}_hac{h}_x"]
                    n = len(x)
                    bands = ward_bands(n, world)
                    for res in results:
                        labels, computed, assembled, received = res[("labels", chunk, layout, tag, h)]
                        assert np.array_equal(labels, gold[f"{tag}_hac{h}_labels"]), (chunk, layout, tag, h)
                        q = res["rank"]
                        plan = ward_chunks(n, bands[q], bands[q + 1], chunk)
                        assert computed == [c for c in plan if c[1] > c[0]]      # this rank's band only, chunk by chunk
                        assert len(plan) > 1 or 8 * band_pairs(n, bands[q], bands[q + 1]) <= chunk
                        if q != 0:
                            assert assembled == [] and received == []
                            continue
                        # rank 0 takes the peers' chunks round robin: chunk k of every rank before chunk k + 1 of any
                        plans = [ward_chunks(n, bands[r], bands[r + 1], chunk) for r in range(world)]
                        order = ward_receive_order(plans)
                        assert received == [(r, band_pairs(n, a, b)) for r, a, b in order if b > a and a < n - 1]
                        assert sorted(order) == sorted((r, a, b) for r in range(1, world) for a, b in plans[r])
                        (D,) = assembled
                        if layout == "square":
                            assert D.shape == (n, n) and np.array_equal(D, W.pdist_square(x))
                        else:
                            assert np.array_equal(D, pdist(x.astype(np.float64)))


def test_rows_that_differ_between_ranks_raise_before_any_band_is_sent(group_results):
    _, results = group_results
    for res in results:
        msg, bands, assembled = res["mismatch"]
        assert "disagree on rows" in msg and bands == [] and assembled == 0


def test_a_chain_failure_on_rank_0_raises_on_every_rank(group_results):
    _, results = group_results
    for res in results:
        assert "ward_labels on rank 0" in res["chain_failure"] and "ALQ_ERR_NUMERIC" in res["chain_failure"]


def test_too_few_or_non_finite_rows_raise_value_error_on_every_rank(group_results):
    _, results = group_results
    for res in results:
        assert "NaN or infinity" in res["value_errors"][0] and "cannot extract 20 clusters" in res["value_errors"][1]


@pytest.mark.parametrize("n", [2, 63, 64, 65, 1000, 115846])
def test_ward_bands_cover_the_pairs_in_equal_shares_on_tile_rows(n):
    from active_learning_b200.sharding import band_pairs, ward_bands, ward_chunks
    total = n * (n - 1) // 2
    for world in range(1, 9):
        b = ward_bands(n, world)
        assert len(b) == world + 1 and b[0] == 0 and b[-1] == n
        assert all(lo <= hi for lo, hi in zip(b, b[1:]))
        assert all(c % 64 == 0 for c in b[1:-1])
        assert sum(band_pairs(n, lo, hi) for lo, hi in zip(b, b[1:])) == total
        for lo, hi in zip(b, b[1:]):
            assert abs(band_pairs(n, lo, hi) * world - total) <= 64 * n * world, (n, world, b)
            for cap in (8, 8 * 5000, 1 << 30):
                plan = ward_chunks(n, lo, hi, cap)
                assert [a for a, _ in plan] + [hi] == [lo] + [c for _, c in plan]      # consecutive, covering
                assert all(c > a and (c - a == 1 or band_pairs(n, a, c) * 8 <= cap) for a, c in plan)


def test_ward_receive_order_is_round_robin_over_the_peers():
    """Chunk k of every peer comes before chunk k + 1 of any (so before chunk k + 2, which a peer with two buffers
    cannot compute before its chunk k is received), each peer's chunks in its sending order, rank 0's own not at all."""
    from active_learning_b200.sharding import ward_bands, ward_chunks, ward_receive_order
    for n, world, cap in ((328, 3, 8 * 700), (1000, 8, 8 * 5000), (80000, 8, 1 << 30), (70, 8, 8 * 50), (500, 1, 64)):
        b = ward_bands(n, world)
        plans = [ward_chunks(n, b[r], b[r + 1], cap) for r in range(world)]
        order = ward_receive_order(plans)
        assert sorted(order) == sorted((r, *c) for r in range(1, world) for c in plans[r])
        index = {(r, *c): k for r in range(1, world) for k, c in enumerate(plans[r])}
        ks = [index[o] for o in order]
        assert ks == sorted(ks)                                           # round by round
        for r in range(1, world):
            assert [o[1:] for o in order if o[0] == r] == plans[r]
        if world == 8 and n == 80000:
            assert [o[0] for o in order[:7]] == list(range(1, 8))


def test_group_layout_counts_the_staging_only_for_the_square_matrix():
    from active_learning_b200._lib import AlqError
    from active_learning_b200.engine import Engine
    from active_learning_b200.sharding import ward_group_layout
    n, staging = 115846, 4 << 30
    cond, sq = Engine.ward_condensed_bytes(n), Engine.ward_bytes(n)
    assert ward_group_layout(n, cond, staging) == "condensed"              # the one-GPU limit, no staging taken off
    assert ward_group_layout(n, sq + staging - 1, staging) == "condensed"
    assert ward_group_layout(n, sq + staging, staging) == "square"
    with pytest.raises(AlqError, match=f"{cond}"):
        ward_group_layout(n, cond - 1, staging)
