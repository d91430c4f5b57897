"""K7 split by bands of rows (MarginClusteringSampler on several GPUs), timed on one H100 with CUDA events.

    python tools/ward_sharded_time.py [--n 80000] [--d 2048] [--repeats 3] [--parent-src DIR] [--out FILE]

At n x d (default 80 000 x 2 048, post-ReLU Gaussian rows) it reports, each as min / median / max over --repeats:
  * full K7 (alq_pdist_f64_condensed, alq_pdist_f64) against the one-band path ShardGroup.ward_labels takes with one
    rank: the band [0, n) in chunks of sharding.WARD_CHUNK_BYTES (alq_pdist_f64_condensed_rows), straight into the
    vector (condensed) or through a staging buffer and alq_pdist_f64_expand into the matrix (square, expand included);
  * the expand kernel alone over those chunks, as a fraction of the H100 SXM's 3.35 TB/s (8 bytes read and 16 written
    per pair);
  * each band of ward_bands(n, G), G = 2, 4, 8, computed one after another on this GPU: the slowest band's time over
    the mean is the balance of the plan (on G GPUs the slowest band bounds K7);
  * with --parent-src (the csrc/ directory of another revision, compiled here with this build's nvcc flags), that
    library's full K7 in both layouts against this build's, alternating within each repetition (and which of the two
    goes first, from one repetition to the next).
Several GPUs are not measured by this tool.  Prints the card's name and power limit first, then one JSON line per
measurement.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_TBPS = 3.35               # H100 SXM data sheet


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:    # noqa: BLE001
        return f"unknown ({e})"


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def stats(ms):
    ms = sorted(ms)
    return {"min_ms": round(ms[0], 2), "median_ms": round(ms[len(ms) // 2], 2), "max_ms": round(ms[-1], 2)}


def build_parent(src):
    """libalq.so from another revision's csrc/ (same nvcc flags as this build), in a temporary directory."""
    import concurrent.futures
    from active_learning_b200 import build as B
    nvcc = B.shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    out = tempfile.mkdtemp(prefix="alq_parent_")
    cus = sorted(f for f in os.listdir(src) if f.endswith(".cu"))
    objs = [os.path.join(out, f[:-3] + ".o") for f in cus]
    with concurrent.futures.ThreadPoolExecutor(max_workers=8) as ex:
        list(ex.map(lambda fo: subprocess.run([nvcc, *B.NVCC_FLAGS, "-c", os.path.join(src, fo[0]), "-o", fo[1]],
                                              check=True, capture_output=True), zip(cus, objs)))
    lib = os.path.join(out, "libalq.so")
    subprocess.run([nvcc, "-shared", *B.GENCODE, "-o", lib, *objs], check=True)
    return lib


class ParentK7:
    """alq_pdist_f64 / alq_pdist_f64_condensed of another libalq.so, on its own context."""

    def __init__(self, path):
        from active_learning_b200 import _lib
        self.lib = C.CDLL(path)
        for name in ("alq_create", "alq_pdist_f64", "alq_pdist_f64_condensed"):
            res, args = _lib.SIGNATURES[name]
            fn = getattr(self.lib, name)
            fn.restype, fn.argtypes = res, args
        self.h = C.c_void_p()
        assert self.lib.alq_create(C.byref(self.h), torch.cuda.current_device()) == 0

    def pdist(self, x, out, condensed):
        s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        n, d = x.shape
        if condensed:
            rc = self.lib.alq_pdist_f64_condensed(self.h, C.c_void_p(x.data_ptr()), n, d, d, C.c_void_p(out.data_ptr()), s)
        else:
            rc = self.lib.alq_pdist_f64(self.h, C.c_void_p(x.data_ptr()), n, d, d, C.c_void_p(out.data_ptr()), n, s)
        assert rc == 0, rc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=80000)
    ap.add_argument("--d", type=int, default=2048)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--parent-src", default=None)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from active_learning_b200 import sharding
    from active_learning_b200.engine import Engine
    n, d = args.n, args.d
    eng = Engine()
    parent = ParentK7(build_parent(args.parent_src)) if args.parent_src else None
    results = [{"card": card(), "torch_device": torch.cuda.get_device_name(), "n": n, "d": d}]
    print(json.dumps(results[0]), flush=True)

    def emit(rec):
        results.append(rec)
        print(json.dumps(rec), flush=True)

    g = torch.Generator(device="cuda").manual_seed(n)
    x = torch.relu(torch.randn(n, d, device="cuda", generator=g))
    m = n * (n - 1) // 2
    chunks = sharding.ward_chunks(n, 0, n, sharding.WARD_CHUNK_BYTES)
    piece = max(sharding.band_pairs(n, a, b) for a, b in chunks)
    eng.pdist(x[:512], condensed=True)                                 # warm-up: module load, first launches
    eng.pdist(x[:512])

    # -- condensed: full K7 against the one-band path (chunks straight into the vector) --------------------------------
    D = torch.empty(m, dtype=torch.float64, device="cuda")
    full, band, par = [], [], []
    for rep in range(args.repeats):
        if parent and rep % 2:
            par.append(timed(lambda: parent.pdist(x, D, True)))
        full.append(timed(lambda: eng.pdist(x, out=D, condensed=True)))

        def one_band():
            for a, b in chunks:
                at = sharding.band_pairs(n, 0, a)
                eng.pdist_rows(x, a, b, out=D[at:at + sharding.band_pairs(n, a, b)])
        band.append(timed(one_band))
        if parent and not rep % 2:
            par.append(timed(lambda: parent.pdist(x, D, True)))
    emit({"layout": "condensed", "what": "full K7", **stats(full)})
    emit({"layout": "condensed", "what": "one band, chunked", "chunks": len(chunks), **stats(band)})
    if parent:
        emit({"layout": "condensed", "what": "full K7, parent build", **stats(par)})

    # -- bands of ward_bands(n, G), one after another, into the vector ----------------------------------------------------
    for G in (2, 4, 8):
        bounds = sharding.ward_bands(n, G)
        per = []
        for lo, hi in zip(bounds, bounds[1:]):
            at = sharding.band_pairs(n, 0, lo)
            per.append(min(timed(lambda: eng.pdist_rows(x, lo, hi, out=D[at:at + sharding.band_pairs(n, lo, hi)]))
                           for _ in range(args.repeats)))
        mean = sum(per) / G
        emit({"what": "ward_bands", "G": G, "bounds": bounds, "band_ms": [round(t, 2) for t in per],
              "max_over_mean": round(max(per) / mean, 4)})
    del D
    torch.cuda.empty_cache()

    # -- square: full K7 against the one-band path (chunks through staging + expand) ------------------------------------
    S = torch.empty((n, n), dtype=torch.float64, device="cuda")
    bufs = [torch.empty(piece, dtype=torch.float64, device="cuda") for _ in range(2)]
    full, band, par, expand = [], [], [], []
    for rep in range(args.repeats):
        if parent and rep % 2:
            par.append(timed(lambda: parent.pdist(x, S, False)))
        full.append(timed(lambda: eng.pdist(x, out=S)))

        def one_band_square():
            for k, (a, b) in enumerate(chunks):
                buf = bufs[k % 2][:sharding.band_pairs(n, a, b)]
                eng.pdist_rows(x, a, b, out=buf)
                eng.pdist_expand(buf, n, a, b, S)
        band.append(timed(one_band_square))
        ex = 0.0
        for k, (a, b) in enumerate(chunks):                            # each chunk recomputed, its expand timed alone
            buf = bufs[k % 2][:sharding.band_pairs(n, a, b)]
            eng.pdist_rows(x, a, b, out=buf)
            ex += timed(lambda: eng.pdist_expand(buf, n, a, b, S))
        expand.append(ex)
        if parent and not rep % 2:
            par.append(timed(lambda: parent.pdist(x, S, False)))
    emit({"layout": "square", "what": "full K7", **stats(full)})
    emit({"layout": "square", "what": "one band, chunked, expand included", "chunks": len(chunks), **stats(band)})
    bytes_moved = 24 * m + 8 * n
    emit({"what": "expand alone", **stats(expand), "bytes": bytes_moved,
          "fraction_of_hbm": round(bytes_moved / (min(expand) * 1e-3) / (HBM_TBPS * 1e12), 3)})
    if parent:
        emit({"layout": "square", "what": "full K7, parent build", **stats(par)})
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
