"""The C-ABI boundary: libalq.so loads on a CPU-only box and exports exactly the entry points
include/alq.h declares; the ctypes binding mirrors them.  No compute calls here."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_functions():
    src = open(os.path.join(ROOT, "include", "alq.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return set(re.findall(r"\b(alq_[a-z0-9_]+)\s*\(", src))


def test_library_exports_every_declared_symbol():
    from active_learning_b200 import _lib, build
    if not os.path.exists(_lib.LIB_PATH):
        build.build()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    declared = _header_functions()
    assert len(declared) >= 14
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in alq.h but not exported"


def test_ctypes_binding_mirrors_header():
    from active_learning_b200 import _lib
    assert set(_lib.SIGNATURES) == _header_functions()
    lib = _lib.load()
    assert lib.alq_version() == _lib.ABI_VERSION


def test_greedy_desc_layout_matches_header_field_order():
    from active_learning_b200 import _lib
    src = open(os.path.join(ROOT, "include", "alq.h")).read()
    body = src[src.index("typedef struct alq_greedy_desc {"):src.index("} alq_greedy_desc;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = re.findall(r"(\w+)\s*;", body)
    assert fields == [f[0] for f in _lib.GreedyDesc._fields_]


def test_create_without_gpu_fails_cleanly():
    import torch
    if torch.cuda.is_available():
        return
    from active_learning_b200 import _lib
    lib = _lib.load()
    h = ctypes.c_void_p()
    assert lib.alq_create(ctypes.byref(h), 0) != 0 and not h.value


def _header_prototypes():
    src = open(os.path.join(ROOT, "include", "alq.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    protos = {}
    for ret, name, args in re.findall(r"\b(int64_t|int|void|const char\*)\s+(alq_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", src):
        args = [a.strip() for a in args.split(",") if a.strip() and a.strip() != "void"]
        protos[name] = (ret, args)
    return protos


def test_ctypes_argument_lists_match_the_header_prototypes():
    """Every parameter of every prototype: pointer vs 32-bit vs 64-bit integer must agree with the ctypes argtypes
    (a drifted binding would pass garbage without any error)."""
    from active_learning_b200 import _lib
    protos = _header_prototypes()
    assert set(protos) == set(_lib.SIGNATURES)

    def kind_of_c(decl):
        if "*" in decl:
            return "ptr"
        t = decl.split()[-2] if len(decl.split()) > 1 else decl
        return {"int64_t": "i64", "int32_t": "i32", "int": "i32", "size_t": "i64"}[t]

    def kind_of_ctypes(t):
        if t in (ctypes.c_int64, ctypes.c_size_t):
            return "i64"
        if t in (ctypes.c_int32, ctypes.c_int):
            return "i32"
        return "ptr"                                   # c_void_p, c_char_p, POINTER(...)

    for name, (ret, args) in protos.items():
        restype, argtypes = _lib.SIGNATURES[name]
        assert [kind_of_c(a) for a in args] == [kind_of_ctypes(t) for t in argtypes], name
        assert (restype is None) == (ret == "void"), name


def test_pairwise_leaf_bounds_is_numpys_tree_and_matches_the_host_twin():
    """alq_pairwise_leaf_bounds (host-only, callable without a GPU) against the Python twin used by the shard planner,
    and against NumPy itself: summing float32 leaves left to right in NumPy's own blocking reproduces np.sum bit for bit
    only if the leaves are the real ones."""
    import numpy as np
    from active_learning_b200 import _lib
    from active_learning_b200.sharding import pairwise_leaf_bounds, plan_shards
    lib = _lib.load()
    for n in (1, 7, 128, 129, 1000, 13000, 130000, 130007):
        out = np.empty(n // 64 + 8, dtype=np.int32)
        k = lib.alq_pairwise_leaf_bounds(n, ctypes.c_void_p(out.ctypes.data), len(out))
        twin = pairwise_leaf_bounds(n)
        assert k == len(twin) - 1 and out[:k + 1].tolist() == twin.tolist()
        assert twin[0] == 0 and twin[-1] == n and (np.diff(twin) <= 128).all() and (np.diff(twin) > 0).all()
    assert lib.alq_pairwise_leaf_bounds(1000, ctypes.c_void_p(out.ctypes.data), 2) == -1
    # the tree is NumPy's: fold the leaves' own np.sum values along the recursion and compare with np.sum
    rng = np.random.default_rng(0)
    x = rng.random(130007).astype(np.float32)

    def fold(lo, m):
        if m <= 128:
            return np.sum(x[lo:lo + m])
        half = m // 2
        half -= half % 8
        return np.float32(fold(lo, half) + fold(lo + half, m - half))

    assert fold(0, len(x)) == np.sum(x)
    # shard planner: leaf-aligned cuts, every candidate inside its rank's position range
    cand = np.sort(rng.choice(130000, 80000, replace=False))
    for world in (2, 3, 8):
        off, pos = plan_shards(cand, 130000, world, leaf_aligned=True)
        b = set(pairwise_leaf_bounds(130000).tolist())
        assert all(int(p) in b for p in pos) and off[0] == 0 and off[-1] == len(cand)
        for r in range(world):
            seg = cand[off[r]:off[r + 1]]
            assert len(seg) and seg.min() >= pos[r] and seg.max() < pos[r + 1]
            assert abs(len(seg) - len(cand) / world) < 200
    off, pos = plan_shards(cand, 130000, 4, leaf_aligned=False)
    assert pos is None and off.tolist() == [0, 20000, 40000, 60000, 80000]


def test_leaf_aligned_shards_cut_on_the_librarys_leaf_bounds():
    """plan_shards(..., leaf_aligned=True) for 1..8 ranks: every shard_pos is a leaf boundary of the library's own
    alq_pairwise_leaf_bounds (the one the selection loop checks them against), and shard_off is where each position
    range starts among the candidates, searchsorted(cand_pos, shard_pos)."""
    import numpy as np
    from active_learning_b200 import _lib
    from active_learning_b200.sharding import plan_shards
    lib = _lib.load()
    rng = np.random.default_rng(3)
    for full_n in (1, 2, 128, 129, 1000, 13007, 130000):
        out = np.empty(full_n // 64 + 8, dtype=np.int32)
        k = lib.alq_pairwise_leaf_bounds(full_n, ctypes.c_void_p(out.ctypes.data), len(out))
        bounds = out[:k + 1]
        for n_cand in sorted({1, max(1, full_n // 7), full_n}):
            cand = np.sort(rng.choice(full_n, n_cand, replace=False))
            for world in range(1, 9):
                off, pos = plan_shards(cand, full_n, world, leaf_aligned=True)
                assert len(pos) == world + 1 and pos[0] == 0 and pos[-1] == full_n
                assert np.isin(pos, bounds).all() and (np.diff(pos) >= 0).all(), (full_n, n_cand, world)
                assert off.tolist() == np.searchsorted(cand, pos).tolist(), (full_n, n_cand, world)
