"""Torch-facing wrapper over the C ABI: torch is only the allocator and the stream provider.

Every method takes CUDA tensors (fp32, row-major, contiguous unless noted), passes
``tensor.data_ptr()`` + ``torch.cuda.current_stream()`` to libalq.so and returns CUDA tensors
(or host NumPy arrays where the reference's API hands host lists back).  There is no CPU code
path here: constructing an Engine without a usable GPU + libalq.so raises.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import numpy as np
import torch

from . import _lib
from ._lib import AlqError, GreedyDesc, MODE_ENTROPY, MODE_LEAST_CONFIDENCE, MODE_MARGIN  # noqa: F401


def _ptr(t: Optional[torch.Tensor]):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _f32c(t: torch.Tensor, name: str) -> torch.Tensor:
    if not t.is_cuda:
        raise AlqError(f"{name} must be a CUDA tensor (no CPU fallback)")
    if t.dtype != torch.float32:
        raise AlqError(f"{name} must be float32, got {t.dtype}")
    if t.dim() == 2 and t.stride(1) == 1 and t.stride(0) >= t.shape[1]:
        return t
    return t.contiguous()


def _ld(t: torch.Tensor) -> int:
    return t.stride(0) if t.dim() == 2 and t.shape[0] > 1 else t.shape[-1]


class Engine:
    """One libalq context bound to one CUDA device."""

    def __init__(self, device: Optional[int] = None):
        self.lib = _lib.load()
        if not torch.cuda.is_available():
            raise AlqError("no CUDA device: the acquisition-scoring engine has no CPU fallback")
        self.device_index = torch.cuda.current_device() if device is None else int(device)
        self.device = torch.device("cuda", self.device_index)
        h = C.c_void_p()
        rc = self.lib.alq_create(C.byref(h), self.device_index)
        if rc != 0:
            raise AlqError(f"alq_create(device={self.device_index}) failed with "
                           f"{_lib.ERR_NAMES.get(rc, rc)} (needs an sm_90 GPU: H100)")
        self._h = h

    def close(self):
        if getattr(self, "_h", None):
            self.lib.alq_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- helpers ---------------------------------------------------------------------------------
    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _check(self, rc, what):
        _lib.check(self.lib, self._h, rc, what)

    def comm_init(self, process_group=None, window_bytes: int = 32 << 20):
        """Create this rank's peer-memory window and map every peer's (CUDA IPC over NVLink).  The 64-byte
        handles travel through torch.distributed (plumbing); afterwards the global CoreSet / k-means++ loops
        exchange their per-step winner from inside the kernels, with no host or NCCL call per step."""
        import torch.distributed as dist
        world, rank = dist.get_world_size(process_group), dist.get_rank(process_group)
        if getattr(self, "comm_ready", False):  # idempotent: samplers and benches may both ask for it
            if (world, rank) != (self.world, self.rank):
                raise AlqError("comm_init: engine is already connected to a different process group")
            return self
        handle = (C.c_char * 64)()
        self._check(self.lib.alq_comm_create(self._h, world, rank, int(window_bytes), handle), "alq_comm_create")
        handles = [None] * world
        dist.all_gather_object(handles, bytes(handle.raw), group=process_group)
        blob = b"".join(handles)
        self._check(self.lib.alq_comm_connect(self._h, blob), "alq_comm_connect")
        self.world, self.rank = world, rank
        self.comm_ready = True
        return self

    def set_option(self, key: str, value: int):
        """'k3_impl': 0 auto / 1 fp32 SIMT / 2 wgmma 3xTF32;  'greedy_variant': 0 auto / 1 direct / 2 pipeline / 3 persistent;  'spin_timeout_ms'; 'l2_resident_mb'; 'd2_fast_path'; 'tail_buckets';
        'select_impl': 0 auto / 1 multi-kernel / 2 cluster;  'base_impl': 0 auto / 1 sequential / 2 parallel lists."""
        self._check(self.lib.alq_set_option(self._h, key.encode(), int(value)), "alq_set_option")

    @property
    def launches(self) -> int:
        return int(self.lib.alq_launch_count(self._h))

    # -- K1 / K1b ----------------------------------------------------------------------------------
    def score_softmax(self, logits: torch.Tensor, mode: int, out: Optional[torch.Tensor] = None):
        logits = _f32c(logits, "logits")
        n, c = logits.shape
        scores = out if out is not None else torch.empty(n, dtype=torch.float32, device=logits.device)
        self._check(self.lib.alq_score_softmax(self._h, _ptr(logits), n, c, _ld(logits), mode,
                                               _ptr(scores), self._stream()), "alq_score_softmax")
        return scores

    def select_smallest(self, scores: torch.Tensor, b: int) -> torch.Tensor:
        scores = _f32c(scores, "scores")
        n = scores.numel()
        b = int(b)
        out = torch.empty(b, dtype=torch.int32, device=scores.device)
        self._check(self.lib.alq_select_smallest(self._h, _ptr(scores), n, b, _ptr(out),
                                                 self._stream()), "alq_select_smallest")
        return out

    def uncertainty_tail(self, logits: torch.Tensor, mode: int, b: int, scores_out: Optional[torch.Tensor] = None):
        """K1 + K1b in one call (one launch when the fused path applies): (scores [n], positions [b] int32,
        ascending (score, position))."""
        logits = _f32c(logits, "logits")
        n, c = logits.shape
        scores = scores_out if scores_out is not None else torch.empty(n, dtype=torch.float32, device=logits.device)
        out = torch.empty(int(b), dtype=torch.int32, device=logits.device)
        self._check(self.lib.alq_uncertainty_tail(self._h, _ptr(logits), n, c, _ld(logits), mode, int(b), _ptr(scores), _ptr(out),
                                                  self._stream()), "alq_uncertainty_tail")
        return scores, out

    def uncertainty_tail_timing(self):
        """(stream_ms, kernel_ms) of the last fused tail launch, from in-kernel %globaltimer stamps (synchronises)."""
        torch.cuda.synchronize(self.device)
        ms = (C.c_float * 2)()
        self._check(self.lib.alq_uncertainty_tail_timing(self._h, C.addressof(ms)), "alq_uncertainty_tail_timing")
        return float(ms[0]), float(ms[1])

    def uncertainty_tail_sharded(self, logits: torch.Tensor, mode: int, b: int, row_lo: int, rows_min: int, rows_max: int,
                                 scores_out: Optional[torch.Tensor] = None):
        """K1 + K1b + the cross-GPU exchange in one call (one launch per rank when the fused path applies):
        (scores [n] of this shard, global positions [b] int32 -- identical on every rank).  Collective over comm_init's group."""
        logits = _f32c(logits, "logits")
        n, c = logits.shape
        scores = scores_out if scores_out is not None else torch.empty(max(n, 1), dtype=torch.float32, device=logits.device)
        out = torch.empty(int(b), dtype=torch.int32, device=logits.device)
        self._check(self.lib.alq_uncertainty_tail_sharded(self._h, _ptr(logits), n, c, _ld(logits) if n else c, mode, int(b), int(row_lo),
                                                          int(rows_min), int(rows_max), _ptr(scores), _ptr(out), self._stream()),
                    "alq_uncertainty_tail_sharded")
        return scores, out

    def topb_pack(self, scores: torch.Tensor, pos: torch.Tensor, row_lo: int, b_pad: int,
                  out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Local winners as packed (score key << 32 | global position) int64 words, ~0-padded to b_pad."""
        if out is None:
            out = torch.empty(int(b_pad), dtype=torch.int64, device=scores.device)
        self._check(self.lib.alq_topb_pack(self._h, _ptr(scores), _ptr(pos), pos.numel(), int(row_lo), int(b_pad),
                                           _ptr(out), self._stream()), "alq_topb_pack")
        return out

    def topb_merge(self, keys: torch.Tensor, b: int, list_len: int = 0) -> torch.Tensor:
        """Global positions (int32) of the b smallest packed words, ascending.  list_len > 0: `keys` is a
        concatenation of individually sorted lists of that length (merge by rank counting, no sort)."""
        out = torch.empty(int(b), dtype=torch.int32, device=keys.device)
        self._check(self.lib.alq_topb_merge(self._h, _ptr(keys), keys.numel(), int(list_len), int(b), _ptr(out),
                                            self._stream()), "alq_topb_merge")
        return out

    def topb_exchange(self, scores: torch.Tensor, pos: torch.Tensor, row_lo: int, b: int) -> torch.Tensor:
        """Global top-b over the ranks of the peer-memory group (comm_init): every rank contributes its local winners
        and gets the b global positions (int32, device) -- no NCCL call."""
        out = torch.empty(int(b), dtype=torch.int32, device=scores.device)
        self._check(self.lib.alq_topb_exchange(self._h, _ptr(scores), _ptr(pos), pos.numel(), int(row_lo), int(b),
                                               _ptr(out), self._stream()), "alq_topb_exchange")
        return out

    def comm_check(self):
        """Raises AlqError if an asynchronous peer-window exchange (topb_exchange) timed out waiting for a peer.  Only
        final after the stream the exchange ran on has been synchronised (e.g. by copying its result to the host)."""
        self._check(self.lib.alq_comm_check(self._h), "alq_comm_check")

    def uncertainty_query_host(self, logits_host: torch.Tensor, mode: int, b: int) -> np.ndarray:
        """Host-buffer entry point (H2D + K1 + K1b + D2H inside the library)."""
        if logits_host.is_cuda or logits_host.dtype != torch.float32 or not logits_host.is_contiguous():
            raise AlqError("logits_host must be a contiguous float32 CPU tensor")
        n, c = logits_host.shape
        out = np.empty(int(b), dtype=np.int32)
        with torch.cuda.device(self.device):
            self._check(self.lib.alq_uncertainty_query_host(
                self._h, C.c_void_p(logits_host.data_ptr()), n, c, mode, int(b),
                C.c_void_p(out.ctypes.data)), "alq_uncertainty_query_host")
        return out

    # -- K2 ------------------------------------------------------------------------------------------
    def badge_factors(self, logits: torch.Tensor, batch_size: int, row0: int = 0, n_total: int = 0):
        """row0/n_total: this tensor is rows [row0, row0+n) of a loader pass over n_total rows (sharded pools)."""
        logits = _f32c(logits, "logits")
        n, c = logits.shape
        cpad = (c + 3) & ~3
        a = torch.empty((n, cpad), dtype=torch.float32, device=logits.device)
        an = torch.empty(n, dtype=torch.float32, device=logits.device)
        self._check(self.lib.alq_badge_factors(self._h, _ptr(logits), n, c, _ld(logits), int(batch_size),
                                               int(row0), int(n_total), _ptr(a), cpad, _ptr(an), self._stream()),
                    "alq_badge_factors")
        return a, an

    def badge_pooled_embedding(self, logits: torch.Tensor, emb: torch.Tensor, batch_size: int):
        logits, emb = _f32c(logits, "logits"), _f32c(emb, "emb")
        n, c = logits.shape
        d = emb.shape[1]
        ph = min(16, c)
        pw = 512 // ph
        width = (ph * pw + 3) & ~3     # e.g. C=10 -> 10 x 51 = 510 -> 512: zero columns keep rows 16-byte
        out = torch.zeros((n, width), dtype=torch.float32, device=logits.device)
        self._check(self.lib.alq_badge_pooled_embedding(
            self._h, _ptr(logits), n, c, _ld(logits), int(batch_size), _ptr(emb), d, _ld(emb),
            _ptr(out), width, self._stream()), "alq_badge_pooled_embedding")
        return out

    def row_norm2(self, x: torch.Tensor) -> torch.Tensor:
        x = _f32c(x, "x")
        n, d = x.shape
        out = torch.empty(n, dtype=torch.float32, device=x.device)
        self._check(self.lib.alq_row_norm2(self._h, _ptr(x), n, d, _ld(x), _ptr(out), self._stream()),
                    "alq_row_norm2")
        return out

    # -- K3 ------------------------------------------------------------------------------------------
    def min_dist(self, x, xn, y, yn, xa=None, xan=None, ya=None, yan=None, reduce_max=False,
                 out: Optional[torch.Tensor] = None, accumulate=False) -> torch.Tensor:
        x, y = _f32c(x, "x"), _f32c(y, "y")
        n, d = x.shape
        m = y.shape[0]
        if out is None:
            out = torch.empty(n, dtype=torch.float32, device=x.device)
            accumulate = False
        c = 0
        if xa is not None:
            xa, ya = _f32c(xa, "xa"), _f32c(ya, "ya")
            c = xa.shape[1]
        self._check(self.lib.alq_min_dist(
            self._h, _ptr(x), _ld(x), _ptr(xn), n, _ptr(y), _ld(y), _ptr(yn), m, d,
            _ptr(xa), _ld(xa) if xa is not None else 0, _ptr(xan),
            _ptr(ya), _ld(ya) if ya is not None else 0, _ptr(yan), c,
            int(bool(reduce_max)), int(bool(accumulate)), _ptr(out), self._stream()), "alq_min_dist")
        return out

    def argmin(self, v: torch.Tensor) -> int:
        out = torch.empty(1, dtype=torch.int32, device=v.device)
        self._check(self.lib.alq_argmin(self._h, _ptr(v), v.numel(), _ptr(out), self._stream()),
                    "alq_argmin")
        return int(out.item())

    def ratio_argmin(self, num: Optional[torch.Tensor], den: torch.Tensor, avail: torch.Tensor) -> int:
        """argmin of num / den over rows with avail != 0 (num None = 1): balancing_sampler.py:114-119."""
        den = _f32c(den, "den")
        if num is not None:
            num = _f32c(num, "num")
        if avail.dtype != torch.uint8 or not avail.is_cuda or avail.numel() != den.numel():
            raise AlqError("ratio_argmin: avail must be a CUDA uint8 tensor with one entry per row")
        out = torch.empty(1, dtype=torch.int32, device=den.device)
        self._check(self.lib.alq_ratio_argmin(self._h, _ptr(num), _ptr(den), _ptr(avail.contiguous()), den.numel(), _ptr(out),
                                              self._stream()), "alq_ratio_argmin")
        return int(out.item())

    # -- K6: MASE / BASE ---------------------------------------------------------------------------------
    def class_gap_inv(self, weight: torch.Tensor):
        """Head geometry of the linear classifier: (ginv [c, c padded to x4], gmin [c + 1]) with
        ginv[a, c] = 1 / |w_a - w_c| (inf on the diagonal), gmin[a] = min_c ginv[a, c] and gmin[c] = the spread bound
        of include/alq.h."""
        weight = _f32c(weight, "weight")
        c, m = weight.shape
        ldg = (c + 3) & ~3
        ginv = torch.empty((c, ldg), dtype=torch.float32, device=weight.device)
        gmin = torch.empty(c + 1, dtype=torch.float32, device=weight.device)
        self._check(self.lib.alq_class_gap_inv(self._h, _ptr(weight), c, m, _ld(weight), _ptr(ginv), ldg, _ptr(gmin),
                                               self._stream()), "alq_class_gap_inv")
        return ginv, gmin

    def mase_margins(self, logits: torch.Tensor, gap, want_per_class: bool = False):
        """(min_margin [n], pred [n] int32, radius [n, c] or None): mase_sampler.py:52-80 from the logits slab.
        `gap` is what class_gap_inv returned."""
        logits = _f32c(logits, "logits")
        n, c = logits.shape
        ginv, gmin = gap
        if ginv.shape[0] != c or ginv.shape[1] < c or gmin.numel() != c + 1:
            raise AlqError("mase_margins: the gap table does not match the class count of logits")
        minm = torch.empty(n, dtype=torch.float32, device=logits.device)
        pred = torch.empty(n, dtype=torch.int32, device=logits.device)
        radius = torch.empty((n, c), dtype=torch.float32, device=logits.device) if want_per_class else None
        self._check(self.lib.alq_mase_margins(self._h, _ptr(logits), n, c, _ld(logits), _ptr(ginv), _ld(ginv),
                                              _ptr(gmin), _ptr(minm), _ptr(pred), _ptr(radius), c, self._stream()),
                    "alq_mase_margins")
        return minm, pred, radius

    def base_select(self, min_margin: torch.Tensor, radius: torch.Tensor, pred: torch.Tensor, budget: int):
        """base_sampler.py:22-38 on the device: int32 pool positions in pick order."""
        radius, min_margin = _f32c(radius, "radius"), _f32c(min_margin, "min_margin")
        if pred.dtype != torch.int32 or not pred.is_cuda:
            raise AlqError("base_select: pred must be a CUDA int32 tensor")
        n, c = radius.shape
        out = torch.empty(int(budget), dtype=torch.int32, device=radius.device)
        self._check(self.lib.alq_base_select(self._h, _ptr(min_margin), _ptr(radius), _ld(radius), _ptr(pred.contiguous()),
                                             n, c, int(budget), _ptr(out), self._stream()), "alq_base_select")
        return out

    # -- K4 / K5 ---------------------------------------------------------------------------------------
    def leaf_bounds(self, n: int) -> np.ndarray:
        """Leaf boundaries of NumPy's float32 pairwise summation over n entries (host helper of the library)."""
        cap = int(n) // 64 + 8
        out = np.empty(cap, dtype=np.int32)
        k = int(self.lib.alq_pairwise_leaf_bounds(int(n), C.c_void_p(out.ctypes.data), cap))
        if k < 0:
            raise AlqError(f"alq_pairwise_leaf_bounds({n}) failed")
        return out[:k + 1].copy()

    def greedy_select(self, x: torch.Tensor, xn: torch.Tensor, mind: torch.Tensor,
                      part_off: Sequence[int], budget: Sequence[int],
                      a: Optional[torch.Tensor] = None, an: Optional[torch.Tensor] = None,
                      uniforms: Optional[np.ndarray] = None, vpos: Optional[torch.Tensor] = None,
                      full_n: Optional[Sequence[int]] = None,
                      first_pick: Optional[Sequence[int]] = None, variant: int = 0,
                      time_steps: bool = False, shard_off: Optional[Sequence[int]] = None,
                      shard_pos: Optional[Sequence[int]] = None):
        """Runs the whole selection loop on the device; returns the picked row ids (host int32,
        partition-major, pick order) and, with time_steps, the mean time of a step's streaming phase in ms
        (the full record -- streaming, selection, steps, variant -- is kept in `self.last_greedy_timing`).

        Multi-GPU (comm_init): every tensor is the GLOBAL, replicated array; `shard_off` [world + 1] says which
        rows each rank streams and, for D^2 sampling, `shard_pos` [world + 1] the matching leaf-aligned position
        ranges of the full array (sharding.plan_shards)."""
        x = _f32c(x, "x")
        n, d = x.shape
        part_off_h = np.ascontiguousarray(part_off, dtype=np.int32)
        budget_h = np.ascontiguousarray(budget, dtype=np.int32)
        total = int(budget_h.sum())
        picks = torch.empty(max(total, 1), dtype=torch.int32, device=x.device)
        desc = GreedyDesc()
        desc.struct_size = C.sizeof(GreedyDesc)
        desc.x, desc.ldx, desc.d = x.data_ptr(), _ld(x), d
        if a is not None:
            a = _f32c(a, "a")
            desc.a, desc.lda, desc.c = a.data_ptr(), _ld(a), a.shape[1]
            desc.an = an.data_ptr()
        desc.xn = xn.data_ptr()
        desc.mind = mind.data_ptr()
        desc.n = n
        desc.n_parts = len(budget_h)
        desc.part_off_host = part_off_h.ctypes.data
        desc.budget_host = budget_h.ctypes.data
        keep = [part_off_h, budget_h, picks, x, a]
        if uniforms is not None:
            if vpos is None or full_n is None:
                raise AlqError("D^2 sampling (uniforms given) needs vpos and full_n")
            u = np.ascontiguousarray(uniforms, dtype=np.float64)
            if u.size != total:
                raise AlqError(f"need {total} uniforms, got {u.size}")
            if u.size == 0:
                u = np.zeros(1)
            full_h = np.ascontiguousarray(full_n, dtype=np.int32)
            desc.uniforms_host = u.ctypes.data
            desc.vpos = vpos.data_ptr()
            desc.full_n_host = full_h.ctypes.data
            keep += [u, full_h, vpos]
        if first_pick is not None:
            fp = np.ascontiguousarray(first_pick, dtype=np.int32)
            desc.first_pick_host = fp.ctypes.data
            keep.append(fp)
        if shard_off is not None:
            so = np.ascontiguousarray(shard_off, dtype=np.int32)
            desc.shard_off_host = so.ctypes.data
            keep.append(so)
            if shard_pos is not None:
                sp = np.ascontiguousarray(shard_pos, dtype=np.int32)
                desc.shard_pos_host = sp.ctypes.data
                keep.append(sp)
        desc.picks = picks.data_ptr()
        desc.variant = int(variant)
        ms = (C.c_float * 8)()
        if time_steps:
            desc.step_kernel_ms_host = C.addressof(ms)
        self._check(self.lib.alq_greedy_select(self._h, C.byref(desc), self._stream()), "alq_greedy_select")
        out = picks[:total].cpu().numpy()
        del keep
        if time_steps:
            self.last_greedy_timing = {"stream_ms": float(ms[0]), "select_ms": float(ms[1]), "steps": int(ms[2]),
                                       "variant": int(ms[3]),
                                       "select_phases_ms": [float(ms[i]) for i in range(4, 8)]}
            return out, float(ms[0])
        return out
