"""Ward clustering of MarginClusteringSampler on the H100: K7 (fp64 distances), K8 (nearest-neighbour chain) and the
host cut (alq_ward_labels), timed separately, in either distance layout, and sklearn on the host for comparison.

    python tools/hac_time.py [--sizes 20000 40000 80000 104262 115846] [--layout square|condensed|both]
                             [--sklearn 10000 20000] [--d 2048] [--out FILE]

Rows are post-ReLU Gaussians (what a ResNet's pooled features look like).  After a warm-up at a small size in every
layout, each size runs K7 + K8 `--repeats` times per layout; `both` alternates the square n x n matrix and scipy's
condensed vector within each repetition, in one process.  A layout whose buffer (plus Engine.WARD_HEADROOM_BYTES) does
not fit the free device memory is left out at that size: on an 80 GB card 104 262 and 115 846 rows (ImageNet-LT's
available rows at 10 % labeled, and its whole train set) run condensed only.  The buffer is allocated before each
repetition and freed after it, outside the timed windows; CUDA events around each call give min / median / max.  The K8
window also holds the entry point's host-side set-up before the launch and its 4-byte status read-back after it
(microseconds), so one more repetition per layout under torch.profiler reports both kernels' device time alone.  The
host cut is timed with a wall clock.  K7's rate counts 3 fp64 operations (sub, mul, add) per pair and dimension,
n (n - 1) / 2 * d pairs-dimensions, against the H100 SXM data sheet's FP64 (non-tensor) peak of 34 TFLOP/s -- which
counts an FMA as two operations; K7 may not fuse, so its instruction-bound ceiling is half of that.  K8 is reported per
merge (n - 1 of them) and per chain push (2 (n - 1)).  For the sklearn sizes the GPU labels must equal
AgglomerativeClustering(n_clusters=20).fit(x).labels_.  Prints one JSON line per measurement and the card's name and
power limit first.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

FP64_PEAK_TFLOPS = 34.0       # H100 SXM data sheet, FP64 without tensor cores


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:            # noqa: BLE001
        q = f"unknown ({e})"
    return q


def rows(n, d, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.relu(torch.randn(n, d, device="cuda", generator=g))


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return out, a.elapsed_time(b)


def kernel_ms(prof, name):
    total = 0.0
    for evt in prof.key_averages():
        if name in evt.key:
            total += getattr(evt, "device_time_total", 0.0) or getattr(evt, "cuda_time_total", 0.0)
    return round(total / 1e3, 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="*", default=[20000, 40000, 80000, 104262, 115846])
    ap.add_argument("--layout", choices=["square", "condensed", "both"], default="both")
    ap.add_argument("--sklearn", type=int, nargs="*", default=[10000, 20000])
    ap.add_argument("--d", type=int, default=2048)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from active_learning_b200.engine import Engine, ward_labels_host
    eng = Engine()
    results = [{"card": card(), "torch_device": torch.cuda.get_device_name()}]
    print(json.dumps(results[0]), flush=True)
    layouts = ["square", "condensed"] if args.layout == "both" else [args.layout]

    def alloc(n, layout):
        shape = (n, n) if layout == "square" else (n * (n - 1) // 2,)
        return torch.empty(shape, dtype=torch.float64, device="cuda")

    def tree(x, layout):
        n = x.shape[0]
        dist = alloc(n, layout)
        _, k7_ms = timed(lambda: eng.pdist(x, out=dist, condensed=layout == "condensed"))
        (xy, md), k8_ms = timed(lambda: eng.nn_chain(dist, n))
        del dist
        torch.cuda.empty_cache()
        return xy, md, k7_ms, k8_ms

    x = rows(2000, args.d, 1)                              # warm-up: module load, cluster attributes, scratch
    for layout in layouts:
        tree(x, layout)
    from torch.profiler import ProfilerActivity, profile
    for n in args.sizes:
        x = rows(n, args.d, n)
        free = eng._ward_free_bytes()
        fits = [lay for lay in layouts
                if (eng.ward_bytes(n) if lay == "square" else eng.ward_condensed_bytes(n)) <= free]
        if not fits:
            eng.ward_layout(n, free)                       # raises, naming n and both byte counts
        k7 = {lay: [] for lay in fits}
        k8 = {lay: [] for lay in fits}
        merges = {}
        for _ in range(args.repeats):
            for lay in fits:
                xy, md, k7_ms, k8_ms = tree(x, lay)
                k7[lay].append(k7_ms)
                k8[lay].append(k8_ms)
                merges[lay] = (xy.cpu().numpy(), md.cpu().numpy())
        for lay in fits:
            xy, md = merges[lay]
            t0 = time.perf_counter()
            ward_labels_host(xy, md, n, 20)
            cut_ms = (time.perf_counter() - t0) * 1e3
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                tree(x, lay)
                torch.cuda.synchronize()
            k7_med, k8_med = float(np.median(k7[lay])), float(np.median(k8[lay]))
            ops = 3.0 * n * (n - 1) / 2 * args.d
            rec = {"n": n, "d": args.d, "layout": lay, "repeats": args.repeats,
                   "k7_ms_min_med_max": [round(min(k7[lay]), 2), round(k7_med, 2), round(max(k7[lay]), 2)],
                   "k7_kernel_ms_profiler": kernel_ms(prof, "pdist_f64_kernel"),
                   "k7_tflops": round(ops / k7_med / 1e9, 2),
                   "k7_share_of_fp64_peak": round(ops / k7_med / 1e9 / FP64_PEAK_TFLOPS, 3),
                   "k8_ms_min_med_max": [round(min(k8[lay]), 2), round(k8_med, 2), round(max(k8[lay]), 2)],
                   "k8_kernel_ms_profiler": kernel_ms(prof, "ward_chain_kernel"),
                   "k8_us_per_merge": round(k8_med * 1e3 / (n - 1), 3),
                   "k8_us_per_push": round(k8_med * 1e3 / (2 * (n - 1)), 3),
                   "cut_ms": round(cut_ms, 2)}
            if len(fits) == 2 and lay == "condensed":      # the two layouts walked the same tree
                rec["merges_identical_to_square"] = bool(np.array_equal(xy, merges["square"][0])
                                                         and np.array_equal(md, merges["square"][1]))
            results.append(rec)
            print(json.dumps(rec), flush=True)
        del x
    if args.sklearn:
        from sklearn.cluster import AgglomerativeClustering
    for n in args.sklearn:
        x = rows(n, args.d, n + 1)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        labels = eng.ward_labels(x, 20)                    # the whole product call: allocation, K7, K8, cut
        gpu_ms = (time.perf_counter() - t0) * 1e3
        xh = x.cpu().numpy()
        t0 = time.perf_counter()
        want = AgglomerativeClustering(n_clusters=20).fit(xh).labels_
        sk_s = time.perf_counter() - t0
        rec = {"n": n, "d": args.d, "sklearn_s": round(sk_s, 2), "ward_labels_ms": round(gpu_ms, 2),
               "labels_identical": bool(np.array_equal(labels, want))}
        results.append(rec)
        print(json.dumps(rec), flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(results, fh, indent=1)


if __name__ == "__main__":
    main()
