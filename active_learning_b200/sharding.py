"""Multi-GPU plumbing of the query path: one process per GPU, torch.distributed for the (few,
small) exchanges.  Rows of the scoring kernels and partitions of the partitioned samplers are
independent, so the data path needs no collective; what is exchanged is

  * uncertainty samplers : each rank's local top-B (score, global position) -> one all-gather of
                           G*B 12-byte records -> the same stable merge on every rank;
  * partitioned samplers : partition i runs on rank i % G; the picked row lists are gathered once.

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
