"""ctypes binding of libalq.so (include/alq.h).  No torch types cross this boundary: only
integers, raw device/host pointers and a cudaStream_t.

The library is built in-tree by ``python -m active_learning_b200.build`` (or ``make``).  If it
is missing this module raises: there is no CPU fallback for the scoring path.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libalq.so")

ALQ_OK = 0
ERR_NAMES = {1: "ALQ_ERR_INVALID", 2: "ALQ_ERR_CUDA", 3: "ALQ_ERR_NOMEM", 4: "ALQ_ERR_STATE",
             5: "ALQ_ERR_NUMERIC"}
MODE_MARGIN, MODE_LEAST_CONFIDENCE, MODE_ENTROPY = 0, 1, 2
ABI_VERSION = 10
IPC_HANDLE_BYTES = 64          # ALQ_IPC_HANDLE_BYTES

c_f32p = C.c_void_p
c_i32p = C.c_void_p


class GreedyDesc(C.Structure):
    """struct alq_greedy_desc (include/alq.h)."""
    _fields_ = [
        ("struct_size", C.c_size_t),
        ("x", C.c_void_p), ("ldx", C.c_int64), ("d", C.c_int32),
        ("a", C.c_void_p), ("lda", C.c_int64), ("c", C.c_int32),
        ("xn", C.c_void_p),
        ("an", C.c_void_p),
        ("mind", C.c_void_p),
        ("n", C.c_int64),
        ("n_parts", C.c_int32),
        ("part_off_host", C.c_void_p),
        ("budget_host", C.c_void_p),
        ("uniforms_host", C.c_void_p),
        ("vpos", C.c_void_p),
        ("full_n_host", C.c_void_p),
        ("first_pick_host", C.c_void_p),
        ("picks", C.c_void_p),
        ("variant", C.c_int32),
        ("shard_off_host", C.c_void_p),
        ("shard_pos_host", C.c_void_p),
        ("step_kernel_ms_host", C.c_void_p),
    ]


class BalancingDesc(C.Structure):
    """struct alq_balancing_desc (include/alq.h)."""
    _fields_ = [
        ("struct_size", C.c_size_t),
        ("x", C.c_void_p), ("ldx", C.c_int64), ("d", C.c_int32),
        ("xn", C.c_void_p),
        ("labels", C.c_void_p),
        ("avail", C.c_void_p),
        ("labeled", C.c_void_p),
        ("n", C.c_int64),
        ("c", C.c_int32),
        ("budget", C.c_int64),
        ("mt_key_host", C.c_void_p),
        ("mt_pos_host", C.c_void_p),
        ("picks", C.c_void_p),
        ("n_picks_host", C.c_void_p),
        ("n_balancing_host", C.c_void_p),
        ("shard_off_host", C.c_void_p),
        ("group_free_bytes", C.c_int64),
    ]


# name -> (restype, argtypes); mirrors include/alq.h one to one (tests/test_abi.py checks it)
SIGNATURES = {
    "alq_version": (C.c_int, []),
    "alq_create": (C.c_int, [C.POINTER(C.c_void_p), C.c_int]),
    "alq_destroy": (None, [C.c_void_p]),
    "alq_last_error": (C.c_char_p, [C.c_void_p]),
    "alq_launch_count": (C.c_int64, [C.c_void_p]),
    "alq_set_option": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int64]),
    "alq_comm_create": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_size_t, C.c_void_p]),
    "alq_comm_connect": (C.c_int, [C.c_void_p, C.c_void_p]),
    "alq_comm_destroy": (C.c_int, [C.c_void_p]),
    "alq_score_softmax": (C.c_int, [C.c_void_p, c_f32p, C.c_int64, C.c_int32, C.c_int64, C.c_int32,
                                    c_f32p, C.c_void_p]),
    "alq_select_smallest": (C.c_int, [C.c_void_p, c_f32p, C.c_int64, C.c_int64, c_i32p, C.c_void_p]),
    "alq_uncertainty_tail": (C.c_int, [C.c_void_p, c_f32p, C.c_int64, C.c_int32, C.c_int64, C.c_int32, C.c_int64, c_f32p,
                                       c_i32p, C.c_void_p]),
    "alq_uncertainty_tail_timing": (C.c_int, [C.c_void_p, C.c_void_p]),
    "alq_uncertainty_tail_sharded": (C.c_int, [C.c_void_p, c_f32p, C.c_int64, C.c_int32, C.c_int64, C.c_int32, C.c_int64, C.c_int64,
                                               C.c_int64, C.c_int64, c_f32p, c_i32p, C.c_void_p]),
    "alq_topb_pack": (C.c_int, [C.c_void_p, c_f32p, c_i32p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]),
    "alq_topb_merge": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, c_i32p, C.c_void_p]),
    "alq_topb_exchange": (C.c_int, [C.c_void_p, c_f32p, c_i32p, C.c_int64, C.c_int64, C.c_int64, c_i32p, C.c_void_p]),
    "alq_comm_check": (C.c_int, [C.c_void_p]),
    "alq_uncertainty_query_host": (C.c_int, [C.c_void_p, c_f32p, C.c_int64, C.c_int32, C.c_int32,
                                             C.c_int64, c_i32p]),
    "alq_badge_factors": (C.c_int, [C.c_void_p, c_f32p, C.c_int64, C.c_int32, C.c_int64, C.c_int32,
                                    C.c_int64, C.c_int64, c_f32p, C.c_int64, c_f32p, C.c_void_p]),
    "alq_badge_pooled_embedding": (C.c_int, [C.c_void_p, c_f32p, C.c_int64, C.c_int32, C.c_int64,
                                             C.c_int32, c_f32p, C.c_int32, C.c_int64, c_f32p,
                                             C.c_int64, C.c_void_p]),
    "alq_row_norm2": (C.c_int, [C.c_void_p, c_f32p, C.c_int64, C.c_int32, C.c_int64, c_f32p,
                                C.c_void_p]),
    "alq_min_dist": (C.c_int, [C.c_void_p,
                               c_f32p, C.c_int64, c_f32p, C.c_int64,
                               c_f32p, C.c_int64, c_f32p, C.c_int64, C.c_int32,
                               c_f32p, C.c_int64, c_f32p,
                               c_f32p, C.c_int64, c_f32p, C.c_int32,
                               C.c_int32, C.c_int32, c_f32p, C.c_void_p]),
    "alq_argmin": (C.c_int, [C.c_void_p, c_f32p, C.c_int64, c_i32p, C.c_void_p]),
    "alq_greedy_select": (C.c_int, [C.c_void_p, C.POINTER(GreedyDesc), C.c_void_p]),
    "alq_pairwise_leaf_bounds": (C.c_int64, [C.c_int64, c_i32p, C.c_int64]),
    "alq_ratio_argmin": (C.c_int, [C.c_void_p, c_f32p, c_f32p, C.c_void_p, C.c_int64, c_i32p, C.c_void_p]),
    "alq_class_gap_inv": (C.c_int, [C.c_void_p, c_f32p, C.c_int32, C.c_int32, C.c_int64, c_f32p, C.c_int64,
                                    c_f32p, C.c_void_p]),
    "alq_mase_margins": (C.c_int, [C.c_void_p, c_f32p, C.c_int64, C.c_int32, C.c_int64, c_f32p, C.c_int64,
                                   c_f32p, c_f32p, c_i32p, c_f32p, C.c_int64, C.c_void_p]),
    "alq_base_select": (C.c_int, [C.c_void_p, c_f32p, c_f32p, C.c_int64, c_i32p, C.c_int64, C.c_int32,
                                  C.c_int64, c_i32p, C.c_void_p]),
    "alq_pdist_f64": (C.c_int, [C.c_void_p, c_f32p, C.c_int64, C.c_int32, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]),
    "alq_ward_nn_chain": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, c_i32p, C.c_void_p, C.c_void_p]),
    "alq_pdist_f64_condensed": (C.c_int, [C.c_void_p, c_f32p, C.c_int64, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p]),
    "alq_ward_nn_chain_condensed": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, c_i32p, C.c_void_p, C.c_void_p]),
    "alq_ward_labels": (C.c_int, [c_i32p, C.c_void_p, C.c_int64, C.c_int32, c_i32p]),
    "alq_pdist_f64_condensed_rows": (C.c_int, [C.c_void_p, c_f32p, C.c_int64, C.c_int32, C.c_int64, C.c_int64, C.c_int64,
                                               C.c_void_p, C.c_void_p]),
    "alq_pdist_f64_expand": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_int64,
                                       C.c_void_p]),
    "alq_ward_nn_chain_banded": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, c_i32p, C.c_void_p,
                                           C.c_void_p]),
    "alq_band_alloc": (C.c_int, [C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p), C.c_void_p]),
    "alq_band_open": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]),
    "alq_band_close": (C.c_int, [C.c_void_p, C.c_void_p]),
    "alq_band_free": (C.c_int, [C.c_void_p, C.c_void_p]),
    "alq_vaal_scores": (C.c_int, [C.c_void_p, c_f32p, C.c_int64, C.c_int32, C.c_int64, c_f32p, C.c_int64, c_f32p,
                                  c_f32p, C.c_int64, c_f32p, c_f32p, c_f32p, C.c_int32, c_f32p, c_f32p, C.c_void_p]),
    "alq_class_counts": (C.c_int, [C.c_void_p, c_i32p, C.c_void_p, C.c_int64, C.c_int32, c_i32p, C.c_void_p]),
    "alq_class_pick": (C.c_int, [C.c_void_p, c_i32p, C.c_void_p, C.c_int64, C.c_int32, c_i32p, c_i32p, C.c_int64, c_i32p,
                                 C.c_void_p]),
    "alq_balancing_select": (C.c_int, [C.c_void_p, C.POINTER(BalancingDesc), C.c_void_p]),
    "alq_balancing_table_select": (C.c_int, [C.c_void_p, C.POINTER(BalancingDesc), C.c_void_p]),
    "alq_probcover_graph": (C.c_int, [C.c_void_p, c_f32p, C.c_int64, C.c_int32, C.c_int64, C.c_void_p, c_f32p, c_i32p,
                                      C.c_void_p, c_i32p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "alq_probcover_select": (C.c_int, [C.c_void_p, C.c_void_p, c_i32p, C.c_int64, C.c_void_p, C.c_int64, c_i32p,
                                       C.c_void_p, C.c_void_p]),
    "alq_kmeans_rows": (C.c_int, [C.c_void_p, c_f32p, C.c_int64, C.c_int32, C.c_int64, C.c_int32, c_f32p, c_f32p, c_f32p,
                                  C.c_void_p, C.c_void_p]),
    "alq_kmeans_assign": (C.c_int, [C.c_void_p, c_f32p, c_f32p, c_f32p, C.c_void_p, C.c_int64, C.c_int32, c_f32p, C.c_int32,
                                    c_i32p, C.c_void_p, C.c_void_p]),
    "alq_kmeans_update": (C.c_int, [C.c_void_p, c_f32p, C.c_int64, C.c_int32, c_i32p, C.c_int32, c_f32p, C.c_void_p]),
    "alq_typicality": (C.c_int, [C.c_void_p, c_f32p, C.c_int32, c_i32p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                 c_i32p, C.c_void_p]),
    "alq_kmeans_nearest": (C.c_int, [C.c_void_p, c_f32p, C.c_int64, C.c_int32, c_i32p, c_f32p, C.c_int32, c_i32p,
                                     C.c_void_p]),
    "alq_knn": (C.c_int, [C.c_void_p, c_f32p, C.c_int64, c_f32p, C.c_int64, C.c_int32, C.c_int32, c_i32p, C.c_void_p,
                          C.c_void_p, C.c_void_p]),
    "alq_cal_scores": (C.c_int, [C.c_void_p, c_f32p, C.c_int64, c_f32p, C.c_int64, C.c_int32, c_i32p, C.c_int32,
                                 C.c_void_p, c_f32p, C.c_void_p]),
    "alq_alfamix_rho": (C.c_int, [C.c_void_p, c_f32p, C.c_int64, C.c_int32, c_f32p, C.c_int32, c_f32p, c_f32p, C.c_int32,
                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
}


class AlqError(RuntimeError):
    pass


_lib = None


def load():
    """dlopen libalq.so and attach prototypes.  Raises if the library was not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise AlqError(
            f"{LIB_PATH} not found: build it with `python -m active_learning_b200.build` "
            "(needs nvcc; there is no CPU fallback for the scoring path)")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)   # AttributeError here == header/library skew
        fn.restype = res
        fn.argtypes = args
    if lib.alq_version() != ABI_VERSION:
        raise AlqError(f"libalq.so ABI {lib.alq_version()} != binding ABI {ABI_VERSION}: rebuild")
    _lib = lib
    return lib


def check(lib, ctx, rc, what):
    if rc != ALQ_OK:
        msg = lib.alq_last_error(ctx)
        raise AlqError(f"{what}: {ERR_NAMES.get(rc, rc)}: {msg.decode() if msg else ''}")
