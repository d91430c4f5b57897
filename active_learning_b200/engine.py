"""Torch-facing wrapper over the C ABI: torch is only the allocator and the stream provider.

Every method takes CUDA tensors (fp32, row-major, contiguous unless noted), passes
``tensor.data_ptr()`` + ``torch.cuda.current_stream()`` to libalq.so and returns CUDA tensors
(or host NumPy arrays where the reference's API hands host lists back).  There is no CPU code
path here: constructing an Engine without a usable GPU + libalq.so raises.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional, Sequence

import numpy as np
import torch

from . import _lib
from ._lib import AlqError, GreedyDesc, MODE_ENTROPY, MODE_LEAST_CONFIDENCE, MODE_MARGIN  # noqa: F401
from .sharding import band_pairs


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


def _mask(t, n: int, device: torch.device, method: str, name: str) -> torch.Tensor:
    """t as a contiguous 1-D uint8 view: a uint8 (or bool) CUDA tensor on `device` with n entries, else AlqError."""
    if (not isinstance(t, torch.Tensor) or not t.is_cuda or t.device != device or t.dtype not in (torch.uint8, torch.bool)
            or t.numel() != n):
        raise AlqError(f"{method}: {name} must be a CUDA uint8 (or bool) tensor on {device} with one entry per row "
                       f"({n})")
    return t.contiguous().view(torch.uint8).reshape(-1)


def _i32(t, shape: Sequence[Optional[int]], device: torch.device, method: str, name: str) -> torch.Tensor:
    """t contiguous: an int32 CUDA tensor on `device` of `shape` (None: any extent), else AlqError."""
    if (not isinstance(t, torch.Tensor) or not t.is_cuda or t.device != device or t.dtype != torch.int32
            or t.dim() != len(shape) or any(s is not None and s != e for s, e in zip(shape, t.shape))):
        dims = ", ".join("any" if s is None else str(s) for s in shape)
        raise AlqError(f"{method}: {name} must be an int32 CUDA tensor on {device} of shape [{dims}]")
    return t.contiguous()


def _pad_width(d: int) -> int:
    """d rounded up to a multiple of 4 (at least 4): the tensor maps want 16-byte rows."""
    return max(4, (int(d) + 3) & ~3)


def _pad4(x: torch.Tensor) -> torch.Tensor:
    """x with zero columns up to _pad_width (a zero column changes no distance, norm or dot product)."""
    n, d = x.shape
    dp = _pad_width(d)
    if dp == d:
        return x
    slab = torch.zeros((n, dp), dtype=torch.float32, device=x.device)
    slab[:, :d] = x
    return slab


def _finite_rows(x: torch.Tensor, method: str) -> torch.Tensor:
    """x as float32 CUDA rows padded by _pad4; ValueError (naming `method`) for an empty matrix or a NaN or infinity."""
    x = _f32c(x, "x")
    if x.dim() != 2 or x.shape[0] == 0:
        raise ValueError(f"{method}: need a non-empty [n, d] matrix, got {tuple(x.shape)}")
    if not bool(torch.isfinite(x).all()):
        raise ValueError(f"{method}: the embeddings contain NaN or infinity")
    return _pad4(x)


def _check_fits(engine, method: str, n: int, need: int, what: str, shrink: str):
    """AlqError naming n, the bytes needed (for `what`) and the bytes free when `need` exceeds engine._ward_free_bytes()."""
    free = engine._ward_free_bytes()
    if need > free:
        raise AlqError(f"{method}: n={n} rows need {need} bytes of device memory ({what}); {free} are free; use a "
                       f"smaller {shrink}")


def ward_labels_host(merge_xy: np.ndarray, merge_dist: np.ndarray, n: int, n_clusters: int) -> np.ndarray:
    """alq_ward_labels (host-only, no GPU): K8's discovery-order merge list -> sklearn's labels for n_clusters (int64)."""
    lib = _lib.load()
    xy = np.ascontiguousarray(merge_xy, dtype=np.int32).reshape(-1, 2)
    md = np.ascontiguousarray(merge_dist, dtype=np.float64).reshape(-1)
    n = int(n)
    if xy.shape[0] != n - 1 or md.shape[0] != n - 1:
        raise AlqError(f"ward labels: need {n - 1} merges for {n} rows, got {xy.shape[0]} / {md.shape[0]}")
    if int(n_clusters) > n:
        raise ValueError(f"cannot extract {n_clusters} clusters from a tree with {n} leaves")
    out = np.empty(n, dtype=np.int32)
    rc = lib.alq_ward_labels(C.c_void_p(xy.ctypes.data), C.c_void_p(md.ctypes.data), n, int(n_clusters),
                             C.c_void_p(out.ctypes.data))
    if rc != 0:
        raise AlqError(f"alq_ward_labels(n={n}, n_clusters={n_clusters}) failed with {_lib.ERR_NAMES.get(rc, rc)}")
    return out.astype(np.int64)


class WardBand:
    """One band of Ward's condensed distances in device memory another process can map: from Engine.band_alloc (owned:
    release() frees it) or Engine.band_open (a peer's: release() unmaps it).  `handle` is the 64-byte CUDA IPC handle.
    Exposes __cuda_array_interface__ as a 1-D float64 array of nbytes // 8 entries, so tensor() is a zero-copy view
    (for pdist_rows(..., out=)); the view must not outlive release()."""

    def __init__(self, engine, ptr: int, nbytes: int, handle: bytes, owned: bool):
        self.engine, self.ptr, self.nbytes, self.handle, self.owned = engine, int(ptr), int(nbytes), handle, owned

    @property
    def __cuda_array_interface__(self):
        return {"shape": (self.nbytes // 8,), "typestr": "<f8", "data": (self.ptr, False), "version": 3,
                "strides": None}

    def tensor(self) -> torch.Tensor:
        return torch.as_tensor(self, device=self.engine.device)

    def release(self):
        """Frees (owned) or unmaps (opened) the band; idempotent."""
        if not self.ptr:
            return
        ptr, self.ptr = self.ptr, 0
        e = self.engine
        if self.owned:
            e._check(e.lib.alq_band_free(e._h, C.c_void_p(ptr)), "alq_band_free")
        else:
            e._check(e.lib.alq_band_close(e._h, C.c_void_p(ptr)), "alq_band_close")


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
        self.comm_group = process_group
        self.comm_ready = True
        return self

    def set_option(self, key: str, value: int):
        """'k3_impl': 0 auto / 1 fp32 SIMT / 2 wgmma 3xTF32;  'greedy_variant' (selection loop only): 0 auto / 1 direct / 2 pipeline / 3 persistent;  'spin_timeout_ms'; 'l2_resident_mb'; 'd2_fast_path'; 'tail_buckets';
        'select_impl': 0 auto / 1 multi-kernel / 2 cluster;  'base_impl': 0 auto / 1 sequential / 2 parallel lists;
        'balancing_loop': 0 auto / 1 per-step path / 2 persistent loop K11 / 3 table loop K12 (2, 3: AlqError beyond the limits)."""
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

    # -- K7 / K8: Ward clustering (MarginClusteringSampler) ---------------------------------------------
    WARD_HEADROOM_BYTES = 1 << 30     # the chain scratch, the merge list and whatever else the query holds

    def pdist(self, x: torch.Tensor, out: Optional[torch.Tensor] = None, condensed: bool = False) -> torch.Tensor:
        """K7: scipy's pdist(x, 'euclidean') bit for bit.  By default the n x n fp64 matrix (diagonal 0); with
        condensed=True scipy's own 1-D layout, n (n - 1) / 2 entries with (i, j), i < j, at n i - i (i + 1) / 2 + j - i - 1
        (half the memory; `out` may be longer, its tail is left untouched)."""
        x = _f32c(x, "x")
        n, d = x.shape
        if condensed:
            m = n * (n - 1) // 2
            if out is None:
                out = torch.empty(max(m, 1), dtype=torch.float64, device=x.device)[:m]
            if not out.is_cuda or out.dtype != torch.float64 or out.dim() != 1 or out.shape[0] < m or out.stride(0) != 1:
                raise AlqError(f"pdist: a condensed out must be a contiguous 1-D float64 CUDA tensor of at least {m} "
                               f"entries")
            if m:
                self._check(self.lib.alq_pdist_f64_condensed(self._h, _ptr(x), n, d, _ld(x), _ptr(out), self._stream()),
                            "alq_pdist_f64_condensed")
            return out
        if out is None:
            out = torch.empty((n, n), dtype=torch.float64, device=x.device)
        if out.dtype != torch.float64 or out.dim() != 2 or out.shape[0] < n or out.shape[1] < n or out.stride(1) != 1:
            raise AlqError("pdist: out must be a row-major float64 CUDA tensor of at least n x n")
        self._check(self.lib.alq_pdist_f64(self._h, _ptr(x), n, d, _ld(x), _ptr(out), out.stride(0), self._stream()),
                    "alq_pdist_f64")
        return out

    def pdist_rows(self, x: torch.Tensor, row_lo: int, row_hi: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """K7 over a band of rows: the entries (i, j), row_lo <= i < row_hi, j > i, of pdist(x, condensed=True), bit for
        bit, as one contiguous fp64 vector (the band's slice of scipy's vector).  `out` may be longer; its tail is left
        untouched.  An empty band returns an empty vector."""
        x = _f32c(x, "x")
        n, d = x.shape
        lo, hi = int(row_lo), int(row_hi)
        if not 0 <= lo <= hi <= n:
            raise AlqError(f"pdist_rows: rows [{lo}, {hi}) are not a band of {n} rows")
        m = band_pairs(n, lo, hi)
        if out is None:
            out = torch.empty(max(m, 1), dtype=torch.float64, device=x.device)[:m]
        if not out.is_cuda or out.dtype != torch.float64 or out.dim() != 1 or out.shape[0] < m or out.stride(0) != 1:
            raise AlqError(f"pdist_rows: out must be a contiguous 1-D float64 CUDA tensor of at least {m} entries")
        if m:
            self._check(self.lib.alq_pdist_f64_condensed_rows(self._h, _ptr(x), n, d, _ld(x), lo, hi, _ptr(out),
                                                              self._stream()), "alq_pdist_f64_condensed_rows")
        return out

    def pdist_expand(self, rows: torch.Tensor, n: int, row_lo: int, row_hi: int, dist: torch.Tensor) -> torch.Tensor:
        """A band from pdist_rows (rows [row_lo, row_hi) of n) into the square matrix `dist` (row-major fp64, at least
        n x n): both (i, j) and (j, i) of every pair of the band, and 0.0 on the band's diagonal.  Bands covering [0, n)
        give exactly pdist(x).  Returns `dist`."""
        n, lo, hi = int(n), int(row_lo), int(row_hi)
        if not 0 <= lo <= hi <= n:
            raise AlqError(f"pdist_expand: rows [{lo}, {hi}) are not a band of {n} rows")
        m = band_pairs(n, lo, hi)
        if not rows.is_cuda or rows.dtype != torch.float64 or rows.dim() != 1 or rows.shape[0] < m or rows.stride(0) != 1:
            raise AlqError(f"pdist_expand: rows must be a contiguous 1-D float64 CUDA tensor of at least {m} entries")
        if (not dist.is_cuda or dist.dtype != torch.float64 or dist.dim() != 2 or dist.shape[0] < n or dist.shape[1] < n
                or dist.stride(1) != 1 or dist.stride(0) < n):
            raise AlqError("pdist_expand: dist must be a row-major float64 CUDA tensor of at least n x n")
        if hi > lo:
            # the band [n - 1, n) holds no pair, only a diagonal entry: its rows are never read, and an empty tensor's
            # data_ptr is null, which the library refuses -- any device address stands in
            src = _ptr(rows) if m else _ptr(dist)
            self._check(self.lib.alq_pdist_f64_expand(self._h, src, n, lo, hi, _ptr(dist), dist.stride(0),
                                                      self._stream()), "alq_pdist_f64_expand")
        return dist

    @staticmethod
    def condensed_rows(length: int) -> int:
        """n such that n (n - 1) / 2 == length; AlqError if there is none."""
        length = int(length)
        n = (1 + math.isqrt(1 + 8 * length)) // 2 if length >= 0 else 0
        if n < 2 or n * (n - 1) // 2 != length:
            raise AlqError(f"nn_chain: a condensed distance vector has n (n - 1) / 2 entries for some n >= 2, got {length}")
        return n

    def nn_chain(self, dist: torch.Tensor, n: Optional[int] = None):
        """K8: scipy's Ward nn_chain over `dist` (consumed).  (merge_xy [n-1, 2] int32 with x < y, merge_dist [n-1]
        fp64) on the device, in the chain's discovery order.  `dist` is either a row-major float64 CUDA matrix of at
        least n x n (n defaults to its row count) or scipy's condensed vector, a contiguous 1-D float64 CUDA tensor of
        exactly n (n - 1) / 2 entries (n is inferred from its length).  Synchronous; AlqError (ALQ_ERR_NUMERIC) if a scan
        meets no finite distance."""
        if dist.dim() == 1:
            if not dist.is_cuda or dist.dtype != torch.float64 or dist.stride(0) != 1:
                raise AlqError("nn_chain: a condensed dist must be a contiguous 1-D float64 CUDA tensor")
            m = self.condensed_rows(dist.shape[0])
            if n is not None and int(n) != m:
                raise AlqError(f"nn_chain: n={n} does not match a condensed vector of {dist.shape[0]} entries (n={m})")
            n = m
        else:
            if not dist.is_cuda or dist.dtype != torch.float64 or dist.dim() != 2 or dist.stride(1) != 1:
                raise AlqError("nn_chain: dist must be a row-major float64 CUDA matrix")
            n = dist.shape[0] if n is None else int(n)
            if n < 2 or dist.shape[0] < n or dist.shape[1] < n or dist.stride(0) < n:
                raise AlqError(f"nn_chain: need n >= 2 and a matrix of at least n x n, got n={n} for {tuple(dist.shape)} "
                               f"with row stride {dist.stride(0)}")
        xy = torch.empty((max(n - 1, 1), 2), dtype=torch.int32, device=dist.device)
        md = torch.empty(max(n - 1, 1), dtype=torch.float64, device=dist.device)
        if dist.dim() == 1:
            self._check(self.lib.alq_ward_nn_chain_condensed(self._h, _ptr(dist), n, _ptr(xy), _ptr(md), self._stream()),
                        "alq_ward_nn_chain_condensed")
        else:
            self._check(self.lib.alq_ward_nn_chain(self._h, _ptr(dist), n, dist.stride(0), _ptr(xy), _ptr(md),
                                                   self._stream()), "alq_ward_nn_chain")
        return xy[:n - 1], md[:n - 1]

    def nn_chain_banded(self, row_cuts: Sequence[int], bands: Sequence, n: int):
        """K8 over the condensed vector cut into bands of rows (alq_ward_nn_chain_banded): band b holds rows
        [row_cuts[b], row_cuts[b + 1]) as pdist_rows writes them, at bands[b] -- a WardBand (this process's or one opened
        from a peer), a contiguous float64 CUDA tensor of at least the band's entries, or None for a band without pairs.
        Consumed.  The same merge list, bit for bit, as nn_chain over the whole vector; synchronous; AlqError
        (ALQ_ERR_INVALID) for bad cuts or a missing band, (ALQ_ERR_NUMERIC) if a scan meets no finite distance."""
        n = int(n)
        cuts = np.ascontiguousarray([int(c) for c in row_cuts], dtype=np.int64)
        nb = len(cuts) - 1
        if len(bands) != nb or nb < 1:
            raise AlqError(f"nn_chain_banded: {len(cuts)} cuts need {max(nb, 0)} bands, got {len(bands)}")
        ptrs = (C.c_void_p * nb)()
        for b, band in enumerate(bands):
            m = band_pairs(n, cuts[b], cuts[b + 1]) if 0 <= cuts[b] <= cuts[b + 1] <= n else 0
            if band is None:
                continue
            if isinstance(band, WardBand):
                size, ptr = band.nbytes // 8, band.ptr
            elif (band.is_cuda and band.dtype == torch.float64 and band.dim() == 1 and band.stride(0) == 1
                  and band.device == self.device):
                size, ptr = band.shape[0], band.data_ptr()
            else:
                raise AlqError("nn_chain_banded: a band must be a WardBand or a contiguous 1-D float64 tensor on "
                               f"{self.device}")
            if size < m:
                raise AlqError(f"nn_chain_banded: band {b} holds {size} entries, rows [{cuts[b]}, {cuts[b + 1]}) "
                               f"have {m}")
            ptrs[b] = ptr
        xy = torch.empty((max(n - 1, 1), 2), dtype=torch.int32, device=self.device)
        md = torch.empty(max(n - 1, 1), dtype=torch.float64, device=self.device)
        self._check(self.lib.alq_ward_nn_chain_banded(self._h, C.c_void_p(cuts.ctypes.data), ptrs, nb, n, _ptr(xy),
                                                      _ptr(md), self._stream()), "alq_ward_nn_chain_banded")
        return xy[:max(n - 1, 0)], md[:max(n - 1, 0)]

    def band_alloc(self, nbytes: int) -> "WardBand":
        """Device memory for one band of Ward's distances that another process of the group can map (alq_band_alloc:
        a cudaMalloc allocation of its own, outside torch's caching allocator, so call torch.cuda.empty_cache() first if
        the bytes may sit in torch's cache).  AlqError (ALQ_ERR_NOMEM) if the device cannot hold it."""
        nbytes = max(8, int(nbytes))
        p = C.c_void_p()
        handle = (C.c_char * _lib.IPC_HANDLE_BYTES)()
        self._check(self.lib.alq_band_alloc(self._h, nbytes, C.byref(p), handle), "alq_band_alloc")
        return WardBand(self, p.value, nbytes, bytes(handle.raw), owned=True)

    def band_open(self, handle: bytes, nbytes: int) -> "WardBand":
        """Maps a peer's band (its WardBand.handle) into this process: alq_band_open.  Release it with release()."""
        handle = bytes(handle)
        if len(handle) != _lib.IPC_HANDLE_BYTES:
            raise AlqError(f"band_open: a handle has {_lib.IPC_HANDLE_BYTES} bytes, got {len(handle)}")
        p = C.c_void_p()
        self._check(self.lib.alq_band_open(self._h, handle, C.byref(p)), "alq_band_open")
        return WardBand(self, p.value, int(nbytes), handle, owned=False)

    @classmethod
    def ward_bytes(cls, n: int) -> int:
        """Device memory a Ward tree over n rows needs in the square layout: the 8 n^2 distance matrix plus headroom."""
        return 8 * int(n) * int(n) + cls.WARD_HEADROOM_BYTES

    @classmethod
    def ward_condensed_bytes(cls, n: int) -> int:
        """The same in the condensed layout: scipy's 4 n (n - 1) byte distance vector plus headroom."""
        return 4 * int(n) * (int(n) - 1) + cls.WARD_HEADROOM_BYTES

    @classmethod
    def ward_layout(cls, n: int, free_bytes: int) -> str:
        """'square' whenever the n x n matrix fits `free_bytes` (it is the faster layout where both fit; see DESIGN),
        else 'condensed' when the vector does, else AlqError naming n and both byte counts."""
        if cls.ward_bytes(n) <= free_bytes:
            return "square"
        if cls.ward_condensed_bytes(n) <= free_bytes:
            return "condensed"
        raise AlqError(f"ward: n={n} rows need {cls.ward_bytes(n)} bytes of device memory as the n x n matrix (8 n^2) "
                       f"or {cls.ward_condensed_bytes(n)} as scipy's condensed vector (4 n (n - 1)), each with "
                       f"{cls.WARD_HEADROOM_BYTES} headroom; {free_bytes} are free; use a smaller subset_unlabeled")

    def _ward_free_bytes(self) -> int:
        """Device memory a Ward query can take: free on the device plus what torch's allocator caches unused."""
        free, _total = torch.cuda.mem_get_info(self.device)
        return free + torch.cuda.memory_reserved(self.device) - torch.cuda.memory_allocated(self.device)

    def _ward_guard(self, n: int) -> str:
        return self.ward_layout(n, self._ward_free_bytes())

    def ward_tree(self, x: torch.Tensor):
        """scipy.cluster.hierarchy.ward(x)'s merges before its sort: (merge_xy [n-1, 2] int32, merge_dist [n-1] fp64) as
        host arrays, in discovery order.  Checks the device memory first and never attempts an allocation that cannot
        fit; there is no CPU fallback.  The distances are the n x n matrix when it fits and scipy's condensed vector
        (half the bytes) when only that fits; the merges are the same either way.  ValueError for fewer than 2 rows or
        non-finite rows.  The distances are returned to the device before this returns (torch.cuda.empty_cache, which
        also releases the process's other unused cached blocks): at 80 000 rows the matrix is 51.2 GB that the caching
        allocator would otherwise keep."""
        x = _f32c(x, "x")
        n = x.shape[0]
        if n < 2:
            raise ValueError(f"ward needs at least 2 rows, got {n}")
        layout = self._ward_guard(n)
        if not bool(torch.isfinite(x).all()):
            raise ValueError("ward: the embeddings contain NaN or infinity")
        dist = self.pdist(x, condensed=layout == "condensed")
        try:
            xy, md = self.nn_chain(dist, n)
            xy, md = xy.cpu().numpy(), md.cpu().numpy()
        finally:
            del dist
            torch.cuda.empty_cache()
        return xy, md

    def ward_labels(self, x: torch.Tensor, n_clusters: int) -> np.ndarray:
        """labels_ of sklearn's AgglomerativeClustering(n_clusters).fit(x) (Ward linkage, full tree), identical, as a host
        int64 array.  ValueError for fewer rows than clusters or non-finite rows, as sklearn raises."""
        x = _f32c(x, "x")
        n = x.shape[0]
        if n < max(2, int(n_clusters)):
            raise ValueError(f"cannot extract {n_clusters} clusters from {n} rows")
        xy, md = self.ward_tree(x)
        return ward_labels_host(xy, md, n, n_clusters)

    # -- K9: the VAAL discriminator (VAALSampler) ----------------------------------------------------------
    VAAL_HIDDEN = 512

    @classmethod
    def vaal_layers(cls, discriminator):
        """The three Linear layers of the reference's Discriminator (vaal_discriminator.py): `discriminator.net` (or the
        module itself) must be Sequential(Linear(z, 512), ReLU, Linear(512, 512), ReLU, Linear(512, 1), Sigmoid), with
        biases.  AlqError for any other layout: K9 computes exactly this network and nothing else."""
        import torch.nn as nn
        seq = getattr(discriminator, "net", discriminator)
        kinds = (nn.Linear, nn.ReLU, nn.Linear, nn.ReLU, nn.Linear, nn.Sigmoid)
        h = cls.VAAL_HIDDEN
        if not isinstance(seq, nn.Sequential) or len(seq) != len(kinds) or any(type(m) is not k for m, k in zip(seq, kinds)):
            raise AlqError("vaal_scores: the discriminator must be the reference's Sequential(Linear(z, 512), ReLU, "
                           "Linear(512, 512), ReLU, Linear(512, 1), Sigmoid)")
        l1, l2, l3 = seq[0], seq[2], seq[4]
        shapes = [(l1.out_features, h), (l2.in_features, h), (l2.out_features, h), (l3.in_features, h), (l3.out_features, 1)]
        if any(a != b for a, b in shapes) or any(lin.bias is None for lin in (l1, l2, l3)):
            raise AlqError(f"vaal_scores: the discriminator's Linear layers must be z -> {h} -> {h} -> 1 with biases")
        return l1, l2, l3

    def vaal_scores(self, mu: torch.Tensor, discriminator, return_logits: bool = False):
        """K9: p[i] = discriminator(mu[i, :z]) for the reference's Discriminator (vaal_layers), as a CUDA float32 vector
        (and the pre-sigmoid logits with return_logits).  `mu` is a CUDA float32 [n, >= z] matrix; rows whose leading
        dimension or base address does not suit the tensor-memory loads are copied into a padded slab first."""
        l1, l2, l3 = self.vaal_layers(discriminator)
        mu = _f32c(mu, "mu")
        z = l1.in_features
        if mu.dim() != 2 or mu.shape[1] < z:
            raise AlqError(f"vaal_scores: mu must be [n, >= {z}], got {tuple(mu.shape)}")
        n, zp, dev = mu.shape[0], (z + 3) & ~3, mu.device
        ld = _ld(mu)
        if n and (ld % 4 or mu.data_ptr() % 16):
            slab = torch.zeros((n, zp), dtype=torch.float32, device=dev)
            slab[:, :z] = mu[:, :z]
            mu, ld = slab, zp

        def dev32(t):
            return t.detach().to(device=dev, dtype=torch.float32).contiguous()

        w1 = torch.zeros((self.VAAL_HIDDEN, zp), dtype=torch.float32, device=dev)
        w1[:, :z] = dev32(l1.weight)
        b1, w2, b2 = dev32(l1.bias), dev32(l2.weight), dev32(l2.bias)
        w3, b3 = dev32(l3.weight).reshape(-1), dev32(l3.bias).reshape(-1)
        p = torch.empty(n, dtype=torch.float32, device=dev)
        logits = torch.empty(n, dtype=torch.float32, device=dev) if return_logits else None
        self._check(self.lib.alq_vaal_scores(self._h, _ptr(mu), n, z, ld, _ptr(w1), zp, _ptr(b1), _ptr(w2), w2.shape[1],
                                             _ptr(b2), _ptr(w3), _ptr(b3), self.VAAL_HIDDEN, _ptr(p), _ptr(logits),
                                             self._stream()), "alq_vaal_scores")
        return (p, logits) if return_logits else p

    # -- K10: per-class counts and class-balanced picks (BalancedRandomSampler) -----------------------------
    CLASS_MAX = 32768      # ALQ_CLASS_MAX of include/alq.h

    def _class_inputs(self, labels: torch.Tensor, avail: torch.Tensor, what: str):
        labels = _i32(labels, (None,), self.device, what, "labels")
        return labels, _mask(avail, labels.numel(), self.device, what, "avail")

    def class_counts(self, labels: torch.Tensor, avail: torch.Tensor, num_classes: int) -> torch.Tensor:
        """K10: counts[c] = number of rows with avail != 0 and labels == c, as a CUDA int32 [num_classes] tensor.
        AlqError (ALQ_ERR_INVALID, naming the row) if an available row's label is outside [0, num_classes).
        Synchronises the stream once."""
        labels, avail = self._class_inputs(labels, avail, "class_counts")
        c = int(num_classes)
        if not 1 <= c <= self.CLASS_MAX:
            raise AlqError(f"class_counts: num_classes={c} outside [1, {self.CLASS_MAX}]")
        counts = torch.empty(c, dtype=torch.int32, device=labels.device)
        self._check(self.lib.alq_class_counts(self._h, _ptr(labels), _ptr(avail), labels.numel(), c, _ptr(counts),
                                              self._stream()), "alq_class_counts")
        return counts

    def class_pick(self, labels: torch.Tensor, avail: torch.Tensor, k, perm) -> torch.Tensor:
        """K10: for each class c ascending with k[c] > 0, the perm-th available rows of class c (ascending row order), for
        the k[c] entries of perm that belong to c (perm concatenates the classes' prefixes, classes ascending).  Returns
        a CUDA int32 [sum(k)] tensor; an entry is -1 where its rank is not below the class's count.  `k` and `perm` are
        host or device integer sequences; host ones travel in one copy.  Asynchronous."""
        labels, avail = self._class_inputs(labels, avail, "class_pick")
        dev = labels.device

        def host(x):
            return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)

        k_h, perm_h = host(k).reshape(-1), host(perm).reshape(-1)
        c, b = k_h.size, perm_h.size
        if not 1 <= c <= self.CLASS_MAX:
            raise AlqError(f"class_pick: {c} class budgets, need 1 .. {self.CLASS_MAX}")
        for name, a in (("k", k_h), ("perm", perm_h)):
            if a.size and (a.dtype.kind not in "iu" or a.min() < 0 or a.max() >= 2 ** 31):
                raise AlqError(f"class_pick: {name} must hold non-negative int32 values")
        if int(k_h.sum()) != b:
            raise AlqError(f"class_pick: sum(k) = {int(k_h.sum())} but perm has {b} entries")
        both = torch.from_numpy(np.concatenate([k_h, perm_h]).astype(np.int32)).to(dev, non_blocking=False)
        out = torch.empty(b, dtype=torch.int32, device=dev)
        self._check(self.lib.alq_class_pick(self._h, _ptr(labels), _ptr(avail), labels.numel(), c, _ptr(both),
                                            C.c_void_p(both.data_ptr() + 4 * c), b, _ptr(out), self._stream()),
                    "alq_class_pick")
        return out

    # -- K11: BalancingSampler's whole query -----------------------------------------------------------
    def balancing_select(self, emb: torch.Tensor, xn: torch.Tensor, labels: torch.Tensor, avail: torch.Tensor,
                         labeled: torch.Tensor, num_classes: int, budget: int, shard_off: Optional[Sequence[int]] = None):
        """K11: balancing_sampler.py:58-134 in one persistent launch.  `emb` [n, d] float32 (d and the leading dimension
        multiples of 4), `xn` = row_norm2(emb), `labels` int32 [n], `avail` / `labeled` uint8 (or bool) [n], all on this
        device.  The random steps draw from NumPy's global RandomState exactly as `np.random.choice` would: the state is
        taken from np.random.get_state() and the final one written back with set_state (has_gauss and cached_gaussian
        unchanged).  Returns (picks: host int64 array in pick order, balancing steps), or None when the per-step path
        must run instead (option "balancing_loop" = 1 or 3, or auto beyond the loop's limits; nothing is drawn then).
        AlqError for bad inputs, for a labeled or available row whose label is outside [0, num_classes), and, under
        balancing_loop = 2, for a shape beyond the limits (the message names the limit).

        Sharded (comm_init): every tensor is the GLOBAL array, replicated on every rank, and `shard_off` [world + 1] says
        which rows each rank streams (e.g. ShardGroup.row_range's bounds).  Collective: every rank calls it with the same
        inputs, which one small all_gather_object checks first (sharding.balancing_agreement: AlqError on every rank on a
        mismatch, before any launch).  Every rank returns the same picks, steps and MT19937 state as one GPU would."""
        return self._balancing_call("balancing_select", self.lib.alq_balancing_select, emb, xn, labels, avail, labeled,
                                    num_classes, budget, shard_off)

    def balancing_table_select(self, emb: torch.Tensor, xn: torch.Tensor, labels: torch.Tensor, avail: torch.Tensor,
                               labeled: torch.Tensor, num_classes: int, budget: int,
                               shard_off: Optional[Sequence[int]] = None):
        """K12: the same query, arguments and contract as `balancing_select`, over an incremental row x class table of
        fp64 dot products with the class sums instead of centres in shared memory, so it runs at ImageNet-LT's 1 000
        classes of 2 048 dimensions.  Returns None under option "balancing_loop" = 1 or 2, or under auto beyond its
        limits (shared memory for the per-class tables, rows per CTA segment, counts plus budget below 2^24, the table
        and the per-CTA class sums in free device memory); AlqError naming the limit under balancing_loop = 3.  Sharded
        as `balancing_select`; each rank then holds the table rows of its own shard only, and the memory limit is
        checked against the least free device memory of the group, gathered with the input check."""
        return self._balancing_call("balancing_table_select", self.lib.alq_balancing_table_select, emb, xn, labels, avail,
                                    labeled, num_classes, budget, shard_off)

    def _balancing_call(self, name, fn, emb, xn, labels, avail, labeled, num_classes, budget, shard_off=None):
        """Checks the arguments of K11 / K12 (messages start with `name`), runs `fn` with NumPy's MT19937 state and
        writes the state back; None when the call declined."""
        emb = _f32c(emb, "emb")
        if emb.dim() != 2:
            raise AlqError(f"{name}: emb must be [n, d]")
        n, d = emb.shape
        dev = emb.device
        if n >= 2 ** 31:
            raise AlqError(f"{name}: n={n} rows, need n < 2^31")
        if not isinstance(xn, torch.Tensor) or not xn.is_cuda or xn.dtype != torch.float32 or xn.numel() != n:
            raise AlqError(f"{name}: xn must be a CUDA float32 tensor with one entry per row")
        labels = _i32(labels, (n,), self.device, name, "labels")
        masks = [_mask(avail, n, self.device, name, "avail"), _mask(labeled, n, self.device, name, "labeled")]
        c, budget = int(num_classes), int(budget)
        if not 1 <= c <= self.CLASS_MAX:
            raise AlqError(f"{name}: num_classes={c} outside [1, {self.CLASS_MAX}]")
        if budget < 0:
            raise AlqError(f"{name}: budget={budget} is negative")
        if emb.shape[1] % 4 or _ld(emb) % 4 or emb.data_ptr() % 16:
            raise AlqError(f"{name}: emb needs d and its leading dimension multiples of 4 and a 16-byte aligned base")
        xn = xn.contiguous().reshape(-1)
        so, free_min = None, 0
        if shard_off is not None:
            from .sharding import balancing_agreement
            if not getattr(self, "comm_ready", False):
                raise AlqError(f"{name}: a sharded call (shard_off) needs comm_init first")
            so = np.ascontiguousarray(shard_off, dtype=np.int32).reshape(-1)
            if so.size != self.world + 1:
                raise AlqError(f"{name}: shard_off needs {self.world + 1} offsets for a group of {self.world}, got {so.size}")
            free = torch.cuda.mem_get_info(self.device)[0] if name == "balancing_table_select" else 0
            free_min = balancing_agreement("alq_" + name, (n, d), c, budget, so, labels, masks[0], masks[1], free,
                                           self.comm_group)
        sname, key, pos, has_gauss, cached = np.random.get_state()
        key = np.array(key, dtype=np.uint32)
        pos_c, n_picks, n_bal = C.c_int32(int(pos)), C.c_int64(0), C.c_int64(0)
        picks = torch.empty(max(budget, 1), dtype=torch.int32, device=dev)
        desc = _lib.BalancingDesc()
        desc.struct_size = C.sizeof(_lib.BalancingDesc)
        desc.x, desc.ldx, desc.d = emb.data_ptr(), _ld(emb), d
        desc.xn, desc.labels = xn.data_ptr(), labels.data_ptr()
        desc.avail, desc.labeled = masks[0].data_ptr(), masks[1].data_ptr()
        desc.n, desc.c, desc.budget = n, c, budget
        desc.mt_key_host = key.ctypes.data
        desc.mt_pos_host = C.addressof(pos_c)
        desc.picks = picks.data_ptr()
        desc.n_picks_host, desc.n_balancing_host = C.addressof(n_picks), C.addressof(n_bal)
        if so is not None:
            desc.shard_off_host, desc.group_free_bytes = so.ctypes.data, int(free_min)
        self._check(fn(self._h, C.byref(desc), self._stream()), "alq_" + name)
        if n_picks.value < 0:
            return None
        np.random.set_state((sname, key, int(pos_c.value), has_gauss, cached))
        return picks[:n_picks.value].cpu().numpy().astype(np.int64), int(n_bal.value)

    # -- K13 / K14: ProbCover ---------------------------------------------------------------------------
    PROBCOVER_HEADROOM_BYTES = 1 << 30   # K14's scratch and whatever else the query holds next to the edges

    @classmethod
    def probcover_bytes(cls, nnz: int) -> int:
        """Device memory the columns of a delta-ball graph with nnz edges need: 4 nnz plus headroom."""
        return 4 * int(nnz) + cls.PROBCOVER_HEADROOM_BYTES

    def probcover_graph(self, x: torch.Tensor, delta: float):
        """K13: the delta-ball graph of the L2-normalised rows of x [n, d] (float32, CUDA) as CSR: (row_ptr int64 [n + 1],
        cols int32 [nnz], recheck) with an edge (i, j) iff scipy's fp64 euclidean distance of the normalised fp32 rows is
        < delta, every row's columns ascending, (i, j) and (j, i) both stored.  `recheck` is the number of pairs the
        tensor-core screen left to the exact recomputation.  ValueError for n = 0, a delta that is not finite and > 0, or
        non-finite rows, before anything runs; AlqError naming n, nnz and the bytes when the edges do not fit in the free
        device memory, checked after the count and before the fill."""
        delta = float(delta)
        if not (math.isfinite(delta) and delta > 0):
            raise ValueError(f"probcover: delta must be finite and > 0, got {delta}")
        x = _finite_rows(x, "probcover")
        n, dp = x.shape
        nt = (n + 127) // 128
        xhat = torch.empty((n, dp), dtype=torch.float32, device=x.device)
        tile = torch.empty(n * nt, dtype=torch.int32, device=x.device)
        row_ptr = torch.empty(n + 1, dtype=torch.int64, device=x.device)
        dh, nnz, rech = C.c_double(delta), C.c_int64(0), C.c_int64(0)
        self._check(self.lib.alq_probcover_graph(self._h, _ptr(x), n, dp, _ld(x), C.byref(dh), _ptr(xhat), _ptr(tile),
                                                 _ptr(row_ptr), None, C.byref(nnz), C.byref(rech), self._stream()),
                    "alq_probcover_graph")
        _check_fits(self, "probcover", n, self.probcover_bytes(nnz.value), f"4 nnz for nnz={nnz.value} edges at "
                    f"delta={delta}, with {self.PROBCOVER_HEADROOM_BYTES} headroom", "delta or subset_unlabeled")
        cols = torch.empty(max(nnz.value, 1), dtype=torch.int32, device=x.device)
        self._check(self.lib.alq_probcover_graph(self._h, None, n, dp, dp, C.byref(dh), _ptr(xhat), _ptr(tile),
                                                 _ptr(row_ptr), _ptr(cols), C.byref(nnz), C.byref(rech), self._stream()),
                    "alq_probcover_graph")
        return row_ptr, cols[:nnz.value], int(rech.value)

    def probcover_select(self, row_ptr: torch.Tensor, cols: torch.Tensor, labeled: torch.Tensor, budget: int):
        """K14: the greedy coverage picks over probcover_graph's CSR: each step takes the lowest row of the largest number
        of uncovered rows in its ball and covers them, starting from the balls of the rows with labeled != 0 covered, and
        stops early when nothing uncovered is left.  Returns (picks: host int64 array in pick order, greedy steps)."""
        n = row_ptr.numel() - 1
        if row_ptr.dtype != torch.int64 or cols.dtype != torch.int32 or not row_ptr.is_cuda or not cols.is_cuda:
            raise AlqError("probcover_select: row_ptr (int64) and cols (int32) must be CUDA tensors")
        lab = _mask(labeled, n, self.device, "probcover_select", "labeled")
        budget = int(budget)
        row_ptr, cols = row_ptr.contiguous(), cols.contiguous()
        picks = torch.empty(max(budget, 1), dtype=torch.int32, device=row_ptr.device)
        # an empty cols tensor has a null data pointer, which the library refuses: any device address stands in
        cp = _ptr(cols) if cols.numel() else _ptr(row_ptr)
        steps = C.c_int64(0)
        self._check(self.lib.alq_probcover_select(self._h, _ptr(row_ptr), cp, n, _ptr(lab), budget,
                                                  _ptr(picks), C.byref(steps), self._stream()), "alq_probcover_select")
        return picks[:steps.value].cpu().numpy().astype(np.int64), int(steps.value)

    # -- K22 / K23: MaxHerding --------------------------------------------------------------------------
    HERDING_ROW_BYTES = 4 + 8 + 1 + 12 + 2   # per row: m, the gain, the candidate flag, S's entry, labeled + avail

    @classmethod
    def herding_bytes(cls, n: int, d: int) -> int:
        """Device memory a MaxHerding query over n rows of width d needs: the 4 n^2 fp32 kernel matrix, xhat (4 n dp, dp
        = d padded to a multiple of 4), the per-row arrays of the greedy and Ward's headroom."""
        n = int(n)
        return 4 * n * n + 4 * n * _pad_width(d) + cls.HERDING_ROW_BYTES * n + cls.WARD_HEADROOM_BYTES

    def herding_guard(self, n: int, d: int):
        """AlqError naming n, the bytes needed and the bytes free when herding_bytes(n, d) does not fit the device."""
        _check_fits(self, "maxherding", n, self.herding_bytes(n, d), f"the 4 n^2 kernel matrix, xhat of width {d} and "
                    f"{self.WARD_HEADROOM_BYTES} headroom", "subset_unlabeled")

    def herding_kernel(self, xhat: torch.Tensor, sigma: float) -> torch.Tensor:
        """K22: the Gaussian kernel matrix K [n, n] (float32 CUDA) of the rows of xhat [n, d] (float32 CUDA):
        K_ij = fl32(exp(-(s_ij / q))), s_ij the exact fp64 squared distance (K7's pair arithmetic), q = 2 sigma^2 in fp64.
        Exactly symmetric, diagonal 1.  ValueError for a bad sigma (maxherding.herding_q); AlqError when the matrix does
        not fit (herding_guard, before any allocation) or for a row with a NaN or infinite entry."""
        from .query_strategies.maxherding import herding_q
        q = herding_q(sigma)
        x = _f32c(xhat, "xhat")
        if x.dim() != 2 or x.shape[0] == 0:
            raise AlqError(f"herding_kernel: need a non-empty [n, d] matrix, got {tuple(x.shape)}")
        n, d = x.shape
        self.herding_guard(n, d)
        out = torch.empty((n, n), dtype=torch.float32, device=x.device)
        qh = C.c_double(q)
        self._check(self.lib.alq_herding_kernel(self._h, _ptr(x), n, d, _ld(x), C.byref(qh), _ptr(out), n,
                                                self._stream()), "alq_herding_kernel")
        return out

    def herding_select(self, K: torch.Tensor, labeled: torch.Tensor, avail: torch.Tensor, budget: int):
        """K23: the greedy coverage picks over herding_kernel's matrix, starting from the rows with labeled != 0 and
        choosing among the rows with avail != 0 (uint8 or bool CUDA masks, one entry per row).  Returns (picks: host int64
        array in pick order, min(budget, available rows) long; m: float32 CUDA [n], the final per-row maxima; the sum
        over the steps of the rows each pick changed)."""
        n = K.shape[0] if K.dim() == 2 else -1
        if (not K.is_cuda or K.dtype != torch.float32 or K.dim() != 2 or K.shape[1] != n or K.stride(1) != 1
                or K.stride(0) < n):
            raise AlqError("herding_select: K must be a square row-major float32 CUDA matrix")
        masks = [_mask(labeled, n, self.device, "herding_select", "labeled"),
                 _mask(avail, n, self.device, "herding_select", "avail")]
        budget = int(budget)
        picks = torch.empty(max(budget, 1), dtype=torch.int32, device=K.device)
        m = torch.empty(n, dtype=torch.float32, device=K.device)
        steps, sum_s = C.c_int64(0), C.c_int64(0)
        self._check(self.lib.alq_herding_select(self._h, _ptr(K), n, K.stride(0), _ptr(masks[0]), _ptr(masks[1]), budget,
                                                _ptr(picks), _ptr(m), C.byref(steps), C.byref(sum_s), self._stream()),
                    "alq_herding_select")
        return picks[:steps.value].cpu().numpy().astype(np.int64), m, int(sum_s.value)

    @staticmethod
    def herding_release():
        """Return the query's kernel matrix to the device (torch.cuda.empty_cache, as ward_tree does): the caching
        allocator would otherwise keep its 4 n^2 bytes."""
        torch.cuda.empty_cache()

    # -- K24 / K25 / K26: BAIT --------------------------------------------------------------------------------
    BAIT_MAX_CLASSES = 16      # K26 keeps each row's C x C forms in shared memory and C accumulators in registers

    @classmethod
    def bait_bytes(cls, n: int, c: int, d: int) -> int:
        """Device memory a BAIT query over n rows with C classes and D features needs: the dense A, F and scratch at
        8 dim^2 each (dim = C D), plus the two per-row C x C forms at 8 n C^2 each."""
        dim = int(c) * int(d)
        return 3 * 8 * dim * dim + 2 * 8 * int(n) * int(c) * int(c)

    def bait_guard(self, n: int, c: int, d: int):
        """AlqError naming C, D, the bytes needed and the bytes free when bait_bytes(n, C, D) does not fit the device, or
        C is outside [2, BAIT_MAX_CLASSES]; before anything is allocated."""
        c, d = int(c), int(d)
        _check_fits(self, "bait", n, self.bait_bytes(n, c, d), f"C={c} classes x D={d} features: A, F and scratch at "
                    f"8 (C D)^2 each, the per-row forms at 8 n C^2 each", "model (C D) or subset_unlabeled")
        if not 2 <= c <= self.BAIT_MAX_CLASSES:
            raise AlqError(f"bait: C={c} classes outside [2, {self.BAIT_MAX_CLASSES}] (D={d})")

    def _bait_rows(self, logits: torch.Tensor, emb: torch.Tensor, method: str):
        zl, h = _f32c(logits, "logits").contiguous(), _f32c(emb, "emb").contiguous()
        if zl.dim() != 2 or h.dim() != 2 or zl.shape[0] != h.shape[0] or zl.shape[0] == 0:
            raise AlqError(f"{method}: need logits [n, C] and emb [n, D] with n >= 1, got {tuple(zl.shape)} and "
                           f"{tuple(h.shape)}")
        return zl, h

    def bait_fisher(self, logits: torch.Tensor, emb: torch.Tensor):
        """K24: (p, F): p float64 CUDA [n, C] the fp64 softmax of logits [n, C], F float64 CUDA [C D, C D] the pool's mean
        Fisher (1/n) sum_x (diag p_x - p_x p_x^T) (x) h_x h_x^T of the raw embeddings emb [n, D] (both float32 CUDA),
        exactly symmetric.  bait_guard runs first; AlqError (ALQ_ERR_NUMERIC) for a row with a NaN or infinity."""
        zl, h = self._bait_rows(logits, emb, "bait_fisher")
        (n, c), d = zl.shape, h.shape[1]
        self.bait_guard(n, c, d)
        p = torch.empty((n, c), dtype=torch.float64, device=zl.device)
        F = torch.empty((c * d, c * d), dtype=torch.float64, device=zl.device)
        self._check(self.lib.alq_bait_fisher(self._h, _ptr(zl), n, c, c, _ptr(h), d, _ptr(p), _ptr(F), self._stream()),
                    "alq_bait_fisher")
        return p, F

    def bait_init(self, emb: torch.Tensor, F: torch.Tensor, lamb: float):
        """K25: (A, At, Gt) from A = I / lamb: A float64 CUDA [C D, C D], and per row of emb [n, D] the C x C forms
        At_x = |h_x|^2 / lamb I and Gt_x[a, b] = h_x^T F_ab h_x / lamb^2 (float64 CUDA [n, C, C])."""
        from .query_strategies.bait import bait_lamb
        lamb = bait_lamb(lamb)
        h = _f32c(emb, "emb").contiguous()
        dim = F.shape[0] if F.dim() == 2 else -1
        if (h.dim() != 2 or not F.is_cuda or F.dtype != torch.float64 or F.shape != (dim, dim) or not F.is_contiguous()
                or dim % h.shape[1]):
            raise AlqError(f"bait_init: need emb [n, D] and a contiguous float64 F [C D, C D], got {tuple(h.shape)} and "
                           f"{tuple(F.shape)}")
        n, d = h.shape
        c = dim // d
        A = torch.empty_like(F)
        At = torch.empty((n, c, c), dtype=torch.float64, device=F.device)
        Gt = torch.empty_like(At)
        lh = C.c_double(lamb)
        self._check(self.lib.alq_bait_init(self._h, _ptr(h), n, c, d, _ptr(F), C.byref(lh), _ptr(A), _ptr(At), _ptr(Gt),
                                           self._stream()), "alq_bait_init")
        return A, At, Gt

    def bait_select(self, emb: torch.Tensor, p: torch.Tensor, F: torch.Tensor, state, lab_pos, cand_pos, budget: int,
                    phase_ms: Optional[np.ndarray] = None):
        """K26: BAIT's picks over the rows of emb [n, D] with bait_fisher's p and F and bait_init's state (A, At, Gt,
        consumed): the rows lab_pos absorbed in order, then T = min(2 budget, len(cand_pos)) forward picks among cand_pos
        (ascending positions) and T - budget backward removals (spec: tests/bait_oracle.py).  Returns (picks: host int64
        array, the remaining list in forward-pick order; the forward picks [T], host int64; the forward scores [T] and
        backward scores [T - budget] of the chosen rows, float64 host arrays).  phase_ms, a float32 host array of 3, receives the device milliseconds of the
        absorption, the forward and the backward pass."""
        A, At, Gt = state
        if phase_ms is not None and (phase_ms.dtype != np.float32 or phase_ms.size < 3 or not phase_ms.flags.c_contiguous):
            raise AlqError("bait_select: phase_ms must be a contiguous float32 host array of at least 3 entries")
        h = _f32c(emb, "emb").contiguous()
        n, d = h.shape
        c = p.shape[1] if p.dim() == 2 else -1
        dim = c * d
        for name, t, shape in (("p", p, (n, c)), ("F", F, (dim, dim)), ("A", A, (dim, dim)), ("At", At, (n, c, c)),
                               ("Gt", Gt, (n, c, c))):
            if not t.is_cuda or t.dtype != torch.float64 or tuple(t.shape) != shape or not t.is_contiguous():
                raise AlqError(f"bait_select: {name} must be a contiguous float64 CUDA tensor of shape {shape}")
        lab = torch.as_tensor(np.asarray(lab_pos, dtype=np.int32), device=h.device)
        cand = np.asarray(cand_pos, dtype=np.int64)
        if len(cand) and (np.any(np.diff(cand) <= 0) or cand[0] < 0 or cand[-1] >= n):
            raise AlqError("bait_select: cand_pos must be ascending pool positions")
        cand_t = torch.as_tensor(cand.astype(np.int32), device=h.device)
        budget = int(budget)
        T = min(2 * budget, len(cand))
        picks = torch.empty(max(budget, 1), dtype=torch.int32, device=h.device)
        fwd_list = torch.empty(max(T, 1), dtype=torch.int32, device=h.device)
        fwd = torch.empty(max(T, 1), dtype=torch.float64, device=h.device)
        bwd = torch.empty(max(T - budget, 1), dtype=torch.float64, device=h.device)
        k = C.c_int64(0)
        self._check(self.lib.alq_bait_select(self._h, _ptr(h), _ptr(p), n, c, d, _ptr(F), _ptr(A), _ptr(At), _ptr(Gt),
                                             _ptr(lab) if len(lab) else None, len(lab),
                                             _ptr(cand_t) if len(cand) else None, len(cand), budget, _ptr(picks),
                                             C.byref(k), _ptr(fwd_list), _ptr(fwd), _ptr(bwd),
                                             None if phase_ms is None else phase_ms.ctypes.data_as(C.c_void_p),
                                             self._stream()), "alq_bait_select")
        return (picks[:k.value].cpu().numpy().astype(np.int64), fwd_list[:T].cpu().numpy().astype(np.int64),
                fwd[:T].cpu().numpy(), bwd[:max(T - budget, 0)].cpu().numpy())

    # -- K15 / K16 / K17: TypiClust ----------------------------------------------------------------------
    KMEANS_MAX_ITER = 100

    def normalize(self, x: torch.Tensor) -> torch.Tensor:
        """The rows of x [n, d] L2-normalised exactly as probcover_graph normalises them, padded with zero columns to a
        multiple of 4: xhat [n, dp] float32.  ValueError for n = 0 or non-finite rows."""
        return self._kmeans_rows(_finite_rows(x, "normalize"), True)[0]

    def _kmeans_rows(self, x: torch.Tensor, normalise: bool):
        """(xhat, hi, lo, nrm2): K15's row operands; with normalise, xhat = the normalised rows of x."""
        n, d = x.shape
        xhat = torch.empty((n, d), dtype=torch.float32, device=x.device) if normalise else x
        hi, lo = torch.empty_like(xhat), torch.empty_like(xhat)
        nrm2 = torch.empty(n, dtype=torch.float64, device=x.device)
        self._check(self.lib.alq_kmeans_rows(self._h, _ptr(x) if normalise else None, n, d, _ld(x), int(normalise),
                                             _ptr(xhat), _ptr(hi), _ptr(lo), _ptr(nrm2), self._stream()),
                    "alq_kmeans_rows")
        return xhat, hi, lo, nrm2

    @staticmethod
    def _kmeans_inputs(xhat: torch.Tensor, centres: torch.Tensor):
        xhat, centres = _f32c(xhat, "xhat").contiguous(), _f32c(centres, "centres").contiguous()
        if xhat.dim() != 2 or centres.dim() != 2 or xhat.shape[1] != centres.shape[1] or xhat.shape[1] % 4:
            raise AlqError(f"kmeans: xhat [n, d] and centres [K, d] with d % 4 == 0, got {tuple(xhat.shape)} and "
                           f"{tuple(centres.shape)}")
        return xhat, centres

    def _assign(self, rows, centres: torch.Tensor, labels: torch.Tensor):
        xhat, hi, lo, nrm2 = rows
        n, d = xhat.shape
        counts = (C.c_int64 * 2)()
        self._check(self.lib.alq_kmeans_assign(self._h, _ptr(xhat), _ptr(hi), _ptr(lo), _ptr(nrm2), n, d, _ptr(centres),
                                               centres.shape[0], _ptr(labels), counts, self._stream()),
                    "alq_kmeans_assign")
        return int(counts[0]), int(counts[1])

    def kmeans_assign(self, xhat: torch.Tensor, centres: torch.Tensor, labels: Optional[torch.Tensor] = None):
        """K15: labels[i] = the lowest c of the minimum of the exact fp64 d2(xhat_i, centres_c) (K7's pair arithmetic).
        `labels` (int32, CUDA) holds the previous labels and is updated in place; None starts from -1.  Returns
        (labels, rows whose label changed, rows the tensor-core screen left to the exact recheck).  The screen's band
        is certified for squared norms in [0, 2] (DESIGN section 4): a row or centre outside it (NaN and infinity
        included) raises AlqError and leaves `labels` untouched; normalised rows and centres that are their means lie
        inside."""
        xhat, centres = self._kmeans_inputs(xhat, centres)
        if labels is None:
            labels = torch.full((xhat.shape[0],), -1, dtype=torch.int32, device=xhat.device)
        elif isinstance(labels, torch.Tensor) and not labels.is_contiguous():
            raise AlqError("kmeans_assign: labels are updated in place and must be contiguous")
        labels = _i32(labels, (xhat.shape[0],), self.device, "kmeans_assign", "labels")
        changed, rech = self._assign(self._kmeans_rows(xhat, False), centres, labels)
        return labels, changed, rech

    def kmeans_update(self, xhat: torch.Tensor, labels: torch.Tensor, centres: torch.Tensor) -> torch.Tensor:
        """K16: centres[c] = fl32(fp64 sum of the rows with label c in ascending row order / their count), in place;
        a cluster with no row keeps its centre.  `centres` must be a contiguous float32 CUDA tensor."""
        xhat = _f32c(xhat, "xhat").contiguous()
        if (centres.dtype != torch.float32 or not centres.is_cuda or not centres.is_contiguous()
                or centres.dim() != 2 or centres.shape[1] != xhat.shape[1]):
            raise AlqError("kmeans_update: centres must be a contiguous float32 CUDA tensor [K, d]")
        n, d = xhat.shape
        labels = _i32(labels, (n,), self.device, "kmeans_update", "labels")
        self._check(self.lib.alq_kmeans_update(self._h, _ptr(xhat), n, d, _ptr(labels), centres.shape[0],
                                               _ptr(centres), self._stream()), "alq_kmeans_update")
        return centres

    def kmeans(self, xhat: torch.Tensor, first_pick: int, uniforms, K: int, max_iter: int = KMEANS_MAX_ITER):
        """k-means of the rows of xhat [n, d] (d % 4 == 0) into K clusters.  Seeding: k-means++ with nothing labeled,
        CoresetQuery's D^2 cold start through greedy_select (centre 0 = row first_pick, then one D^2 draw per uniform,
        K - 1 of them).  Then Lloyd: assign (K15), and while some label changed and fewer than max_iter assignments
        ran, update (K16) and assign again; one 4-byte and one 8-byte copy per assignment.  The rows' squared norms must
        lie in [0, 2] (normalised rows do; AlqError otherwise, from the first assignment).  Returns (labels int32 CUDA
        [n], centres [K, d], assignments run, seed rows)."""
        xhat = _f32c(xhat, "xhat").contiguous()
        n, d = xhat.shape
        K = int(K)
        if not 1 <= K <= n:
            raise ValueError(f"kmeans: K={K} outside [1, n={n}]")
        u = np.zeros(K, dtype=np.float64)
        u[1:] = np.asarray(uniforms, dtype=np.float64).reshape(-1)[:K - 1]
        if np.asarray(uniforms).size != K - 1:
            raise ValueError(f"kmeans: need K - 1 = {K - 1} uniforms, got {np.asarray(uniforms).size}")
        mind = torch.full((n,), float("inf"), dtype=torch.float32, device=xhat.device)
        seeds = self.greedy_select(xhat, self.row_norm2(xhat), mind, [0, n], [K], uniforms=u,
                                   vpos=torch.arange(n, dtype=torch.int32, device=xhat.device), full_n=[n],
                                   first_pick=[int(first_pick)]).astype(np.int64)
        centres = xhat.index_select(0, torch.as_tensor(seeds, device=xhat.device)).contiguous()
        rows = self._kmeans_rows(self._kmeans_inputs(xhat, centres)[0], False)
        labels = torch.full((n,), -1, dtype=torch.int32, device=xhat.device)
        it = 0
        while True:
            changed, _ = self._assign(rows, centres, labels)
            it += 1
            if changed == 0 or it >= int(max_iter):
                return labels, centres, it, seeds
            self.kmeans_update(xhat, labels, centres)

    def typicality(self, xhat: torch.Tensor, rows: torch.Tensor, group_off: Sequence[int], k: int = 20):
        """K17: rows[group_off[g]:group_off[g + 1]] (int32 CUDA row ids of xhat) form group g.  Per listed row, with
        k' = min(k, group size // 2): typicality = 1 / (mean + 1e-5), mean = the ascending fp64 sum of its k' smallest
        exact squared distances to the other rows of its group / k' (0 for a group of one row).  Returns (typicality
        float64 CUDA [len(rows)], host int64 [groups]: the position in rows of each group's largest, lowest on ties).
        k must lie in [1, 32] (AlqError otherwise)."""
        xhat = _f32c(xhat, "xhat").contiguous()
        rows = _i32(rows, (None,), self.device, "typicality", "rows")
        goff = np.ascontiguousarray(group_off, dtype=np.int64)
        if goff.ndim != 1 or len(goff) < 2 or goff[-1] != rows.numel():
            raise AlqError("typicality: group_off must run from 0 to len(rows)")
        g = len(goff) - 1
        typ = torch.empty(max(rows.numel(), 1), dtype=torch.float64, device=xhat.device)
        best = torch.empty(g, dtype=torch.int32, device=xhat.device)
        self._check(self.lib.alq_typicality(self._h, _ptr(xhat), xhat.shape[1], _ptr(rows), C.c_void_p(goff.ctypes.data),
                                            g, int(k), _ptr(typ), _ptr(best), self._stream()), "alq_typicality")
        return typ[:rows.numel()], best.cpu().numpy().astype(np.int64)

    def kmeans_nearest(self, xhat: torch.Tensor, labels: torch.Tensor, centres: torch.Tensor) -> np.ndarray:
        """K21: per cluster c < K the row labeled c with the smallest exact fp64 d2(xhat_i, centres_c) (K7's pair
        arithmetic), the lowest row on ties; -1 for an empty cluster.  Rows labeled outside [0, K) are skipped.  Returns
        host int64 [K]."""
        xhat, centres = self._kmeans_inputs(xhat, centres)
        labels = _i32(labels, (xhat.shape[0],), self.device, "kmeans_nearest", "labels")
        k = centres.shape[0]
        out = torch.empty(max(k, 1), dtype=torch.int32, device=xhat.device)
        self._check(self.lib.alq_kmeans_nearest(self._h, _ptr(xhat), xhat.shape[0], xhat.shape[1], _ptr(labels),
                                                _ptr(centres), k, _ptr(out), self._stream()), "alq_kmeans_nearest")
        return out[:k].cpu().numpy().astype(np.int64)

    # -- K20: ALFA-Mix -------------------------------------------------------------------------------
    def alfamix_rho(self, logits: torch.Tensor, emb: torch.Tensor, anchors: torch.Tensor, weight: torch.Tensor,
                    want_parts: bool = False):
        """K20: ALFA-Mix's closed-form mixing test per row (spec: tests/alfamix_oracle.py).  logits [n, C], emb [n, Dp] and
        anchors [C, Dp] (the raw embeddings and class anchors, zero columns past D), weight [C, D] the linear head, all
        float32 CUDA.  rho_u = sqrt(D) t*_u / R_u, where t*_u is the smallest feature step along the loss gradient that
        changes the predicted class and R_u the largest exact distance to an anchor; row u's mixed features flip its
        prediction at cap eps exactly when rho_u < eps sqrt(D).  Returns rho float64 CUDA [n], or (rho, R^2, t*) with
        want_parts.  AlqError for C < 2, mismatched shapes, or a non-finite entry."""
        zl, z = _f32c(logits, "logits").contiguous(), _f32c(emb, "emb").contiguous()
        a, w = _f32c(anchors, "anchors").contiguous(), _f32c(weight, "weight").contiguous()
        if z.dim() == 2 and a.dim() == 2:
            z, a = _pad4(z), _pad4(a)
        if (zl.dim() != 2 or z.dim() != 2 or a.dim() != 2 or w.dim() != 2 or zl.shape[0] != z.shape[0]
                or zl.shape[1] != w.shape[0] or a.shape[0] != w.shape[0] or a.shape[1] != z.shape[1]
                or w.shape[1] > z.shape[1]):
            raise AlqError(f"alfamix_rho: need logits [n, C], emb [n, Dp], anchors [C, Dp] and weight [C, D <= Dp], got "
                           f"{tuple(zl.shape)}, {tuple(z.shape)}, {tuple(a.shape)} and {tuple(w.shape)}")
        n = zl.shape[0]
        outs = [torch.empty(max(n, 1), dtype=torch.float64, device=zl.device) for _ in range(3 if want_parts else 1)]
        ptrs = [_ptr(t) for t in outs] + [None] * (3 - len(outs))
        self._check(self.lib.alq_alfamix_rho(self._h, _ptr(zl), n, zl.shape[1], _ptr(z), z.shape[1], _ptr(a), _ptr(w),
                                             w.shape[1], *ptrs, self._stream()), "alq_alfamix_rho")
        outs = [t[:n] for t in outs]
        return tuple(outs) if want_parts else outs[0]

    # -- K18 / K19: CAL ------------------------------------------------------------------------------
    def knn(self, x: torch.Tensor, y: torch.Tensor, k: int):
        """K18: the k nearest rows of y [m, d] for every row of x [n, d] (float32 CUDA, d % 4 == 0) by the exact fp64
        squared distance of the raw rows (K7's pair arithmetic), ascending (d2, row of y).  Returns (idx int32 CUDA
        [n, k], d2 float64 CUDA [n, k], rows that took the exact fallback scan); past m entries are -1 / +inf.  AlqError
        for k outside [1, 32], d % 4 != 0, an empty x or y, or a squared row norm that is not finite or above 2^100."""
        x, y = _f32c(x, "x").contiguous(), _f32c(y, "y").contiguous()
        if x.dim() != 2 or y.dim() != 2 or x.shape[1] != y.shape[1]:
            raise AlqError(f"knn: need x [n, d] and y [m, d], got {tuple(x.shape)} and {tuple(y.shape)}")
        n, k = x.shape[0], int(k)
        idx = torch.empty((n, max(k, 1)), dtype=torch.int32, device=x.device)
        d2 = torch.empty((n, max(k, 1)), dtype=torch.float64, device=x.device)
        fallback = C.c_int64(0)
        self._check(self.lib.alq_knn(self._h, _ptr(x), n, _ptr(y), y.shape[0], x.shape[1], k, _ptr(idx), _ptr(d2),
                                     C.byref(fallback), self._stream()), "alq_knn")
        return idx, d2, int(fallback.value)

    def cal_scores(self, cand_logits: torch.Tensor, ref_logits: torch.Tensor, idx: torch.Tensor):
        """K19: CAL's score of every candidate row against its neighbours idx [n, k] (int32 CUDA rows of ref_logits,
        entries outside [0, m) skipped): the mean over the neighbours of KL(softmax(ref) || softmax(cand)) in fp64 (spec:
        tests/cal_oracle.py).  Returns (score float64 CUDA [n], key float32 CUDA [n]), key = -fl32(score) with +0.0 for a
        zero and +NaN for a NaN score, so that select_smallest(key, b) takes the b largest scores, lowest row on ties."""
        zc, zr = _f32c(cand_logits, "cand_logits").contiguous(), _f32c(ref_logits, "ref_logits").contiguous()
        if zc.dim() != 2 or zr.dim() != 2 or zc.shape[1] != zr.shape[1]:
            raise AlqError(f"cal_scores: need logits [n, C] and [m, C], got {tuple(zc.shape)} and {tuple(zr.shape)}")
        n = zc.shape[0]
        idx = _i32(idx, (n, None), self.device, "cal_scores", "idx")
        score = torch.empty(n, dtype=torch.float64, device=zc.device)
        key = torch.empty(n, dtype=torch.float32, device=zc.device)
        self._check(self.lib.alq_cal_scores(self._h, _ptr(zc), n, _ptr(zr), zr.shape[0], zc.shape[1], _ptr(idx),
                                            idx.shape[1], _ptr(score), _ptr(key), self._stream()), "alq_cal_scores")
        return score, key

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
        ranges of the full array (sharding.plan_shards).  After comm_init a call with `shard_off` takes the group path
        whatever the group's size: a group of one rank runs the group path (the window, its ready handshake and tags)
        on this GPU.  Without comm_init, `shard_off=[0, n]` is ignored and any other split is an AlqError."""
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
