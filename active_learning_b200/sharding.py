"""Multi-GPU plumbing of the query path: one process per GPU, torch.distributed for the (few,
small) exchanges.  Rows of the scoring kernels and partitions of the partitioned samplers are
independent, so the data path needs no collective; what is exchanged is

  * uncertainty samplers : each rank's local top-B (score, global position) -> one all-gather of
                           G*B 12-byte records -> the same stable merge on every rank;
  * partitioned samplers : partition i runs on rank i % G; the picked row lists are gathered once;
  * Ward clustering      : K7 by pair-balanced bands of rows (ward_bands), each band sent to rank 0 in chunks, K8 on
                           rank 0, the n labels broadcast back (ShardGroup.ward_labels); when rank 0 cannot hold the
                           distances, each band stays on its rank and K8 reads it through CUDA IPC peer memory.

Works with backend "nccl" (GPU) and "gloo" (the CPU tests of this host logic).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.distributed as dist


def pairwise_leaf_bounds(n: int) -> np.ndarray:
    """Leaf boundaries of NumPy's float32 pairwise summation over n entries (blocks of <= 128, splits at n/2 rounded
    down to a multiple of 8) -- the host twin of the library's alq_pairwise_leaf_bounds (tests pin them together)."""
    out = []

    def rec(lo, m):
        if m <= 128:
            out.append(lo)
            return
        half = m // 2
        half -= half % 8
        rec(lo, half)
        rec(lo + half, m - half)

    rec(0, int(n))
    out.append(int(n))
    return np.asarray(out, dtype=np.int32)


def plan_shards(cand_pos: np.ndarray, full_n: int, world: int, leaf_aligned: bool, leaf_bounds=None):
    """Split the (sorted) candidate rows of one global partition over `world` ranks.

    Returns (shard_off [world + 1] row offsets, shard_pos [world + 1] position offsets or None).  For the arg-max loop
    any split works: equal row counts.  For D^2 sampling every rank must own whole leaves of NumPy's pairwise-sum tree
    over the full (labeled + unlabeled) array, so the cuts are moved to the nearest leaf boundary."""
    n = len(cand_pos)
    if not leaf_aligned:
        return np.asarray([r * n // world for r in range(world + 1)], dtype=np.int32), None
    bounds = pairwise_leaf_bounds(full_n) if leaf_bounds is None else np.asarray(leaf_bounds)
    shard_pos = [0]
    for r in range(1, world):
        target = int(cand_pos[min(n - 1, r * n // world)]) if n else 0
        k = int(np.searchsorted(bounds, target))
        k = min(max(k, 0), len(bounds) - 1)
        if k > 0 and target - bounds[k - 1] < bounds[k] - target:
            k -= 1
        shard_pos.append(max(int(bounds[k]), shard_pos[-1]))
    shard_pos.append(int(full_n))
    shard_pos = np.asarray(shard_pos, dtype=np.int32)
    shard_off = np.searchsorted(np.asarray(cand_pos), shard_pos, side="left").astype(np.int32)
    shard_off[0], shard_off[-1] = 0, n
    return shard_off, shard_pos


def check_replicated(what: str, record: dict, local=None, process_group=None) -> list:
    """A collective call over replicated inputs must see the same inputs on every rank: one all_gather_object of this
    rank's `record` (small host values and digests) together with a rank-local value `local`, and an AlqError naming the
    first field of `record` that differs -- raised on every rank, since every rank compares the same gathered records.
    Returns every rank's `local`, in rank order."""
    from ._lib import AlqError
    out = [None] * dist.get_world_size(process_group)
    dist.all_gather_object(out, (record, local), group=process_group)
    for key in record:
        vals = [r[0].get(key) for r in out]
        if any(v != vals[0] for v in vals[1:]):
            raise AlqError(f"{what}: the ranks disagree on {key} ({vals}); a sharded call needs the same replicated "
                           f"inputs on every rank")
    return [r[1] for r in out]


def digest(*arrays) -> str:
    """sha1 over the bytes of host arrays / tensors (the replicated masks and labels of a collective call)."""
    import hashlib
    h = hashlib.sha1()
    for a in arrays:
        if isinstance(a, torch.Tensor):
            a = a.detach().cpu().contiguous().numpy()
        a = np.ascontiguousarray(a)
        h.update(str(a.dtype).encode() + str(a.shape).encode())
        h.update(a.tobytes())
    return h.hexdigest()


def balancing_agreement(what: str, shape, num_classes: int, budget: int, shard_off, labels, avail, labeled,
                        free_bytes: int = 0, process_group=None) -> int:
    """The host check in front of a sharded BalancingSampler call (K11 / K12): every rank must hold the same n, d, C,
    budget, shard offsets, labels, masks and NumPy MT19937 state, or the ranks would stream different problems and wait
    on each other's words until the timeout.  AlqError on every rank otherwise, before anything runs on the device.
    Returns the least of the ranks' `free_bytes` (K12's table check must decide the same way everywhere)."""
    _, key, pos, _, _ = np.random.get_state()
    record = {"n, d": tuple(int(v) for v in shape), "num_classes": int(num_classes), "budget": int(budget),
              "shard_off": [int(v) for v in shard_off], "labels": digest(labels), "masks": digest(avail, labeled),
              "MT19937 state": digest(np.asarray(key, dtype=np.uint32), np.int64(pos))}
    return min(check_replicated(what, record, int(free_bytes), process_group))


WARD_CHUNK_BYTES = 1 << 30      # largest piece of a K7 band in flight between two ranks (two such buffers per peer)


def band_pairs(n: int, lo: int, hi: int) -> int:
    """Pairs (i, j), lo <= i < hi, j > i, of n rows: the entries rows [lo, hi) occupy in scipy's condensed vector."""
    n, lo, hi = int(n), int(lo), int(hi)
    return (hi - lo) * (n - 1) - (hi * (hi - 1) - lo * (lo - 1)) // 2


def ward_bands(n: int, world: int) -> list:
    """[world + 1] row offsets splitting K7's n (n - 1) / 2 pairs over `world` ranks: from 0 to n, never decreasing,
    interior cuts on multiples of 64 (K7's tile rows stay whole), each band within one tile row (64 n pairs) of an equal
    share.  Row i carries n - 1 - i pairs, so the early bands hold fewer rows.  Bands may be empty for small n."""
    n, world = int(n), int(world)
    total = n * (n - 1) // 2
    cuts = np.arange(0, n + 1, 64, dtype=np.int64)                     # candidate interior cuts
    before = cuts * (n - 1) - cuts * (cuts - 1) // 2                   # pairs above each candidate, increasing
    out = [0]
    for r in range(1, world):
        want = r * total                                               # world * (pairs before the cut), exactly
        k = int(np.searchsorted(before * world, want))
        if k == len(cuts) or (k > 0 and want - before[k - 1] * world <= before[k] * world - want):
            k -= 1
        out.append(max(int(cuts[k]), out[-1]))
    out.append(n)
    return out


def ward_chunks(n: int, lo: int, hi: int, max_bytes: int) -> list:
    """Rows [lo, hi) of a K7 band cut into consecutive (a, b) pieces of at most max_bytes of fp64 pairs each (at least
    one row per piece), cut on multiples of 64 where that keeps a piece non-empty.  Sender and receiver derive the same
    pieces from (n, lo, hi, max_bytes)."""
    out, a = [], int(lo)
    cap = max(1, int(max_bytes) // 8)
    while a < hi:
        b, top = a + 1, int(hi)                                        # largest b with band_pairs(a, b) <= cap
        while b < top:
            mid = (b + top + 1) // 2
            if band_pairs(n, a, mid) <= cap:
                b = mid
            else:
                top = mid - 1
        if b < hi and b - b % 64 > a:
            b -= b % 64
        out.append((a, b))
        a = b
    return out


def ward_receive_order(plan: list) -> list:
    """The order in which rank 0 takes in the peers' chunks: (rank, a, b), round robin over the ranks -- chunk k of every
    rank r >= 1 before chunk k + 1 of any -- so that all peers, each sending its chunks in order from two buffers, make
    progress at the same time.  `plan[r]` is rank r's ward_chunks list."""
    out = []
    for k in range(max((len(p) for p in plan[1:]), default=0)):
        out.extend((r, *plan[r][k]) for r in range(1, len(plan)) if k < len(plan[r]))
    return out


def ward_group_layout(n: int, free_bytes: int, staging_bytes: int) -> str:
    """Rank 0's layout in ShardGroup.ward_labels: the n x n matrix when it fits `free_bytes` together with the staging
    buffers it needs (`staging_bytes`), else scipy's condensed vector (which needs none) when that fits, else the
    AlqError of Engine.ward_layout naming n and both byte counts."""
    from .engine import Engine
    if Engine.ward_bytes(n) + staging_bytes <= free_bytes:
        return "square"
    if Engine.ward_condensed_bytes(n) <= free_bytes:
        return "condensed"
    return Engine.ward_layout(n, free_bytes)          # raises: neither fits


def ward_band_bytes(n: int, world: int) -> list:
    """Bytes of each rank's ward_bands(n, world) band of scipy's condensed vector (8 per pair)."""
    b = ward_bands(n, world)
    return [8 * band_pairs(n, lo, hi) for lo, hi in zip(b, b[1:])]


def ward_group_placement(n: int, free_bytes, staging_bytes: int, distributed: bool = True) -> str:
    """Where ShardGroup.ward_labels keeps the distances, from every rank's free device memory `free_bytes` (rank order):
    ward_group_layout's 'square' or 'condensed' on rank 0 whenever rank 0 fits one of them, else 'distributed' -- each
    rank keeps its own ward_bands band, K8 on rank 0 reads the peers' through peer memory -- when `distributed` (every
    rank's engine has the band calls) and every rank's free memory holds its band plus Engine.WARD_HEADROOM_BYTES, else an
    AlqError naming n, both of rank 0's byte counts and the largest band's."""
    from ._lib import AlqError
    from .engine import Engine
    free_bytes = [int(f) for f in free_bytes]
    try:
        return ward_group_layout(n, free_bytes[0], staging_bytes)
    except AlqError:
        if not distributed:
            raise
    need = [b + Engine.WARD_HEADROOM_BYTES for b in ward_band_bytes(n, len(free_bytes))]
    if all(m <= f for m, f in zip(need, free_bytes)):
        return "distributed"
    raise AlqError(f"ward_labels: n={n} rows need {Engine.ward_bytes(n)} bytes of device memory on rank 0 as the n x n "
                   f"matrix or {Engine.ward_condensed_bytes(n)} as scipy's condensed vector, or, distributed over "
                   f"{len(free_bytes)} ranks, {max(need)} on the rank with the largest band ({max(need) - Engine.WARD_HEADROOM_BYTES} "
                   f"bytes of distances), each with {Engine.WARD_HEADROOM_BYTES} headroom; the ranks have {free_bytes} "
                   f"bytes free; use a smaller subset_unlabeled")


class ShardGroup:
    def __init__(self, process_group=None):
        if not dist.is_initialized():
            raise RuntimeError("torch.distributed is not initialised")
        self.pg = process_group
        self.rank = dist.get_rank(process_group)
        self.world_size = dist.get_world_size(process_group)
        self._buf = {}

    # ---- row sharding (K1 / K2) -----------------------------------------------------------------
    def row_range(self, n, rank=None):
        """Contiguous block of rows owned by `rank`: sizes differ by at most one."""
        r = self.rank if rank is None else rank
        base, rem = divmod(int(n), self.world_size)
        lo = r * base + min(r, rem)
        return lo, lo + base + (1 if r < rem else 0)

    def merge_smallest(self, scores_local, pos_local, row_lo, budget, engine, to_host=True, rendezvous=False):
        """Global `budget` smallest (score, global position) pairs from every rank's local winners.

        scores_local: this rank's score vector; pos_local: its local top-B positions (K1b output);
        row_lo: global position of local row 0.  Each rank packs its winners into 64-bit words
        (order-preserving score key << 32 | global position), ONE all-gather moves G*B words, and
        every rank runs the same device merge: ascending words == ascending (score, position), i.e.
        exactly the single-GPU K1b order.  Only the B winning positions go to the host.

        rendezvous: the peer-window exchange waits for every rank's flag with a bounded spin ("spin_timeout_ms");
        after a phase in which ranks can drift apart by seconds (the per-shard forward pass of a sampler) pass True:
        one barrier first, so that the spin only ever covers kernel-scale skew."""
        b = int(budget)
        if getattr(engine, "comm_ready", False) and b <= 16384:
            # peer-memory windows (Engine.comm_init): packed winners are stored straight into every rank's window
            if rendezvous:
                dist.barrier(group=self.pg)
            try:
                out = engine.topb_exchange(scores_local, pos_local, row_lo, b)
                if not to_host:
                    return out            # asynchronous: a timed-out exchange fills `out` with -1 and is reported by
                                          # Engine.comm_check() / the next exchange
                host = out.cpu().numpy()  # synchronises the stream: the status word is final now
                engine.comm_check()
                return host.astype(np.int64) & 0xFFFFFFFF
            except Exception as exc:      # a peer never raised its flag: fall back to the collective path below
                from ._lib import AlqError
                if not isinstance(exc, AlqError):
                    raise
                self.exchange_failures = getattr(self, "exchange_failures", 0) + 1
        key = (b, scores_local.device)
        if self._buf.get("key") != key:
            self._buf = {"key": key,
                         "mine": torch.empty(b, dtype=torch.int64, device=scores_local.device),
                         "all": torch.empty(b * self.world_size, dtype=torch.int64, device=scores_local.device)}
        mine, allk = self._buf["mine"], self._buf["all"]
        engine.topb_pack(scores_local, pos_local, row_lo, b, out=mine)
        dist.all_gather_into_tensor(allk, mine, group=self.pg)
        out = engine.topb_merge(allk, b, list_len=b)   # G sorted lists -> int32 global positions, on the device
        if not to_host:
            return out
        return out.cpu().numpy().astype(np.int64) & 0xFFFFFFFF

    # ---- variable-length row gathers (plumbing for the global CoreSet / BADGE queries) ----------------
    def all_gather_rows(self, t, counts):
        """Concatenate every rank's [counts[r], D] tensor in rank order.  The counts are known on every
        rank from the (replicated) host bookkeeping, so only padded data travels."""
        width = t.shape[1] if t.dim() == 2 else 1
        cmax = max(int(c) for c in counts) if len(counts) else 0
        pad = torch.zeros((cmax, width), dtype=t.dtype, device=t.device)
        if t.numel():
            pad[:t.shape[0]] = t.reshape(t.shape[0], width)
        out = torch.empty((self.world_size * cmax, width), dtype=t.dtype, device=t.device)
        dist.all_gather_into_tensor(out, pad, group=self.pg)
        parts = [out[r * cmax:r * cmax + int(counts[r])] for r in range(self.world_size)]
        res = torch.cat(parts, dim=0)
        return res if t.dim() == 2 else res.reshape(-1)

    # ---- partition dealing ------------------------------------------------------------------------
    def my_partitions(self, n_parts, rank=None):
        r = self.rank if rank is None else rank
        return [i for i in range(n_parts) if i % self.world_size == r]

    def all_gather_dict(self, mine: dict) -> dict:
        """Union of per-rank {partition: picks} dicts (picks are small int arrays)."""
        payload = {int(k): np.asarray(v).tolist() for k, v in mine.items()}
        out = [None] * self.world_size
        dist.all_gather_object(out, payload, group=self.pg)
        merged = {}
        for d in out:
            for k, v in d.items():
                merged[int(k)] = np.asarray(v, dtype=np.int64)
        return merged

    # ---- Ward clustering (MarginClusteringSampler) ---------------------------------------------------
    def ward_labels(self, x, n_clusters, engine, rows_digest="", layout=None):
        """sklearn's AgglomerativeClustering(n_clusters) labels of the replicated rows x [n, D], on every rank, with K7
        split over the ranks: rank r computes the pairs of its ward_bands(n, G) band (engine.pdist_rows) in chunks of
        at most WARD_CHUNK_BYTES and sends them to rank 0, which assembles the distances (the n x n matrix through
        engine.pdist_expand when it fits, else scipy's condensed vector), runs K8 (engine.nn_chain) and the labelling,
        and broadcasts the labels.  The labels are those of Engine.ward_labels on one GPU.

        Transfer: every peer computes its chunks in order into two buffers and sends each to rank 0 as it is done
        (it waits on the send of two chunks earlier before reusing a buffer).  Rank 0 computes its own band on a side
        stream, so that no receive waits behind it, and takes in the peers' chunks round robin (ward_receive_order):
        condensed, all receives are posted at once, each into its slice of the vector; square, they go through two
        staging buffers, the next chunk received while the previous one is expanded.  An unexpected runtime error in
        the middle of the transfer (the arguments and buffers are checked before it) leaves the other side waiting on
        its send or receive until the process group's timeout; errors before the transfer and in K8 reach every rank.

        Distributed placement (ward_group_placement: only when rank 0 fits neither layout, or when layout="distributed"
        forces it): every rank reserves its band in memory another process can map (engine.band_alloc) before the
        agreement, writes it with one pdist_rows call and synchronises its stream; one all_gather_object exchanges the
        bands' IPC handles; rank 0 maps the peers' bands, runs K8 over all of them in place (engine.nn_chain_banded)
        and the labelling, unmaps them and broadcasts the labels.  Nothing is sent between the GPUs but K8's own peer
        reads and writes.  A peer neither touches nor frees its band until that broadcast has arrived, so the peers wait
        in the broadcast while K8 runs on rank 0: the process group's timeout bounds K8's time.

        `rows_digest` names the pool rows of x (the caller's digest of their positions): the ranks must agree on it.
        ValueError on every rank for fewer than max(2, n_clusters) rows or non-finite rows (sklearn's errors); AlqError on
        every rank, before any distance is sent, if the ranks disagree on n, d, the rows or `layout`, if a rank cannot
        reserve its buffers (or its band), or if the ranks' memory fits no placement; AlqError with rank 0's message if
        K8 fails there or if rank 0 cannot map a peer's band."""
        from ._lib import AlqError
        from .engine import Engine
        n, d = int(x.shape[0]), int(x.shape[1])
        if n < max(2, int(n_clusters)):
            raise ValueError(f"cannot extract {n_clusters} clusters from {n} rows")
        if not bool(torch.isfinite(x).all()):
            raise ValueError("ward: the embeddings contain NaN or infinity")
        if layout not in (None, "distributed"):
            raise ValueError(f"ward_labels: layout must be None or 'distributed', got {layout!r}")
        world, rank = self.world_size, self.rank
        bands = ward_bands(n, world)
        plan = [ward_chunks(n, bands[r], bands[r + 1], WARD_CHUNK_BYTES) for r in range(world)]
        piece = max([band_pairs(n, a, b) for p in plan for a, b in p] + [1])      # entries of the largest chunk
        nbufs = 2 if world == 1 else 4              # square layout on rank 0: its own band's pair, the receiving pair
        staging = nbufs * 8 * piece

        # reserve this rank's buffers (rank 0: D too) before the agreement, so that a failure is raised on every rank
        # there rather than leaving the other ranks waiting on a send or a receive
        # (every rank probes its own free memory: the distributed placement needs each rank's)
        free, err, bufs, hold, band = int(engine._ward_free_bytes()), None, [], [], None
        can_band = hasattr(engine, "nn_chain_banded") and hasattr(engine, "band_alloc")
        layout0 = None
        if rank == 0 and layout is None:
            try:
                layout0 = ward_group_layout(n, free, staging)
            except AlqError:
                pass                                   # neither layout fits: the agreement decides on every rank
        try:
            if layout == "distributed":
                band = self._ward_band(x, n, bands, engine)
            elif rank != 0:
                engine.pdist_rows(x, bands[rank], bands[rank])      # the engine's argument checks, on an empty band
            elif layout0 == "square":
                hold.append(torch.empty((n, n), dtype=torch.float64, device=x.device))
            elif layout0 == "condensed":
                hold.append(torch.empty(n * (n - 1) // 2, dtype=torch.float64, device=x.device))
            if layout is None and (rank != 0 or layout0 == "square"):     # the staging buffers
                bufs = [torch.empty(piece, dtype=torch.float64, device=x.device)
                        for _ in range(2 if rank != 0 else nbufs)]
        except Exception as exc:                       # noqa: BLE001 -- e.g. CUDA out of memory
            err = f"rank {rank}: {type(exc).__name__}: {exc}"
        try:
            record = {"n, d": (n, d), "rows": str(rows_digest), "n_clusters": int(n_clusters), "layout": layout}
            locals_ = check_replicated("ward_labels", record, (free, err, can_band), self.pg)
            errs = [e for _, e, _ in locals_ if e]
            if errs:
                raise AlqError("ward_labels: a rank could not reserve its K7 buffers: " + "; ".join(errs))
            # the same decision (or error) on every rank
            placement = layout or ward_group_placement(n, [f for f, _, _ in locals_], staging,
                                                       all(c for _, _, c in locals_))
            if placement == "distributed":
                if layout is None:
                    # rank 0 fits neither layout: the staging buffers go, each rank reserves its band, and one more
                    # agreement raises a failed reservation on every rank before any band is computed
                    bufs.clear()
                    err = None
                    try:
                        band = self._ward_band(x, n, bands, engine)
                    except Exception as exc:           # noqa: BLE001
                        err = f"rank {rank}: {type(exc).__name__}: {exc}"
                    errs = [e for e in check_replicated("ward_labels", {}, err, self.pg) if e]
                    if errs:
                        raise AlqError("ward_labels: a rank could not reserve its band: " + "; ".join(errs))
                return self._ward_distributed(x, n, int(n_clusters), engine, bands, band)
            layout = placement

            if rank != 0:
                sends = []
                for k, (a, b) in enumerate(plan[rank]):
                    if band_pairs(n, a, b) == 0:
                        continue                       # row n - 1 alone: nothing to send (rank 0 skips it too)
                    if len(sends) >= 2:
                        sends[-2].wait()               # the send of two chunks ago released this buffer
                    buf = bufs[k % 2][:band_pairs(n, a, b)]
                    engine.pdist_rows(x, a, b, out=buf)
                    sends.append(dist.isend(buf, dst=self._global_rank(0), group=self.pg))
                for w in sends[-2:]:
                    w.wait()
                box = [None]
            else:
                box = [self._ward_rank0(x, n, int(n_clusters), engine, layout, plan, bufs, hold)]
        finally:
            bufs.clear()
            on_device = bool(hold) and hold[0].is_cuda
            hold.clear()
            if on_device:
                torch.cuda.empty_cache()               # rank 0's distances go back to the device (as Engine.ward_tree)
            if band is not None:
                band.release()                         # an error before the bands were handed out (else a no-op)
        dist.broadcast_object_list(box, src=self._global_rank(0), group=self.pg)
        msg, labels = box[0]
        if msg is not None:
            raise AlqError(f"ward_labels on rank 0: {msg}")
        return np.asarray(labels).astype(np.int64)

    def _ward_band(self, x, n, bands, engine):
        """This rank's band of the distributed placement, reserved in memory another process can map (None when the
        band holds no pair).  The engine's argument checks run first, on an empty band."""
        from ._lib import AlqError
        if not (hasattr(engine, "nn_chain_banded") and hasattr(engine, "band_alloc")):
            raise AlqError("the engine has no band calls (band_alloc, nn_chain_banded) for the distributed placement")
        lo, hi = bands[self.rank], bands[self.rank + 1]
        engine.pdist_rows(x, lo, lo)
        m = band_pairs(n, lo, hi)
        if not m:
            return None
        if x.is_cuda:
            torch.cuda.empty_cache()                   # the band is the library's cudaMalloc: torch's cache is no use to it
        return engine.band_alloc(8 * m)

    def _ward_distributed(self, x, n, n_clusters, engine, bands, band):
        """The distributed placement of ward_labels, after the agreement: this rank's band from one pdist_rows call,
        the stream synchronised, the handles exchanged, K8 on rank 0 over every band, the labels broadcast.  The band is
        released only after the broadcast (rank 0 has unmapped the peers' bands by then)."""
        from ._lib import AlqError
        rank = self.rank
        box = [None]
        try:
            err = None
            try:
                if band is not None:
                    engine.pdist_rows(x, bands[rank], bands[rank + 1], out=band.tensor())
                    if x.is_cuda:
                        torch.cuda.current_stream(x.device).synchronize()   # K7 is complete before the handle leaves
            except Exception as exc:                   # noqa: BLE001 -- reported by rank 0 on every rank
                err = f"rank {rank}: {type(exc).__name__}: {exc}"
            mine = (err, None if band is None else band.handle, 0 if band is None else band.nbytes)
            shared = [None] * self.world_size
            dist.all_gather_object(shared, mine, group=self.pg)
            if rank == 0:
                box = [self._ward_rank0_banded(n, n_clusters, engine, bands, band, shared)]
            dist.broadcast_object_list(box, src=self._global_rank(0), group=self.pg)
        finally:
            if band is not None:
                band.release()
        msg, labels = box[0]
        if msg is not None:
            raise AlqError(f"ward_labels on rank 0: {msg}")
        return np.asarray(labels).astype(np.int64)

    def _ward_rank0_banded(self, n, n_clusters, engine, bands, band, shared):
        """Rank 0's half of the distributed placement: the peers' bands mapped, K8 over every band, the labels, the
        mappings closed.  Returns (error message or None, labels as int32)."""
        from .engine import ward_labels_host
        errs = [e for e, _, _ in shared if e]
        if errs:
            return "K7 failed: " + "; ".join(errs), None
        opened = []
        try:
            parts = [band]
            for handle, nbytes in ((h, b) for _, h, b in shared[1:]):
                parts.append(None if handle is None else engine.band_open(handle, nbytes))
                if handle is not None:
                    opened.append(parts[-1])
            xy, md = engine.nn_chain_banded(bands, parts, n)          # synchronous: the bands are idle when it returns
            xy = xy.cpu().numpy() if isinstance(xy, torch.Tensor) else np.asarray(xy)
            md = md.cpu().numpy() if isinstance(md, torch.Tensor) else np.asarray(md)
            return None, ward_labels_host(xy, md, n, n_clusters).astype(np.int32)
        except Exception as exc:                       # noqa: BLE001 -- every rank raises rank 0's message
            return f"{type(exc).__name__}: {exc}", None
        finally:
            for b in opened:
                try:
                    b.release()
                except Exception:                      # noqa: BLE001 -- an unmap error must not keep the peers waiting
                    pass

    def _global_rank(self, r):
        return r if self.pg is None else dist.get_global_rank(self.pg, r)

    def _ward_rank0(self, x, n, n_clusters, engine, layout, plan, bufs, hold):
        """Rank 0's half of ward_labels: its own band and every peer's chunks into D = hold[0], K8, the labels.  Returns
        (error message or None, labels as int32); D is released by the caller."""
        import contextlib
        from .engine import ward_labels_host
        D = hold[0]
        cur = torch.cuda.current_stream(D.device) if D.is_cuda else None
        side = torch.cuda.Stream(device=D.device) if D.is_cuda else None
        try:
            square = layout == "square"
            own, recv = bufs[-2:], bufs[:2]             # the same pair when there are no peers
            if side is not None:
                side.wait_stream(cur)                   # x and D are ready on the current stream
            # rank 0's own band, on the side stream: an NCCL receive waits for the stream it is posted from, so on the
            # current stream every receive would wait for the whole band
            with torch.cuda.stream(side) if side is not None else contextlib.nullcontext():
                for j, (a, b) in enumerate(plan[0]):
                    m = band_pairs(n, a, b)
                    if square:
                        buf = own[j % 2][:m]
                        engine.pdist_rows(x, a, b, out=buf)
                        engine.pdist_expand(buf, n, a, b, D)
                    else:
                        at = band_pairs(n, 0, a)
                        engine.pdist_rows(x, a, b, out=D[at:at + m])
            src = {r: self._global_rank(r) for r in range(1, len(plan))}
            order = ward_receive_order(plan)
            if not square:                              # every receive straight into its slice, all in flight at once
                works = []
                for r, a, b in order:
                    m, at = band_pairs(n, a, b), band_pairs(n, 0, a)
                    if m:
                        works.append(dist.irecv(D[at:at + m], src=src[r], group=self.pg))
                for w in works:
                    w.wait()
            else:
                def post(k):
                    """Receive chunk k of the order into staging buffer k % 2 (a pairless chunk, row n - 1 alone, is
                    not sent: only its diagonal entry is written)."""
                    r, a, b = order[k]
                    m = band_pairs(n, a, b)
                    dst = recv[k % 2][:m]
                    return dst, (dist.irecv(dst, src=src[r], group=self.pg) if m else None)

                pending = post(0) if order else None
                for k in range(len(order)):
                    # chunk k + 1 is posted before chunk k is expanded: its buffer's last reader, the expand of chunk
                    # k - 1, is already on the stream ahead of it
                    nxt = post(k + 1) if k + 1 < len(order) else None
                    dst, work = pending
                    if work is not None:
                        work.wait()
                    _, a, b = order[k]
                    engine.pdist_expand(dst, n, a, b, D)
                    pending = nxt
            if side is not None:
                cur.wait_stream(side)
            own, recv = [], []
            bufs.clear()
            xy, md = engine.nn_chain(D, n)
            xy = xy.cpu().numpy() if isinstance(xy, torch.Tensor) else np.asarray(xy)
            md = md.cpu().numpy() if isinstance(md, torch.Tensor) else np.asarray(md)
            return None, ward_labels_host(xy, md, n, n_clusters).astype(np.int32)
        except Exception as exc:                       # noqa: BLE001 -- every rank raises rank 0's message
            return f"{type(exc).__name__}: {exc}", None
        finally:
            if side is not None:
                cur.wait_stream(side)                   # nothing on the side stream outlives D and the buffers
