"""ProbCoverSampler's kernels on the H100: K13 (the delta-ball graph: count pass, memory check, fill pass) and K14 (every
greedy pick in one launch), timed with CUDA events around the Engine calls, with the edges and the pairs K13 sent to the
exact recheck.

    python tools/probcover_time.py [--sizes 20000x512,130000x2048] [--degrees 10,300] [--budget 10000] [--reps 3]

The rows are clustered (cluster centres plus small noise), so that a fixed radius gives a chosen mean degree: clusters
of `degree` rows and delta = 0.8 put every row's ball around its own cluster.  K13's rate is counted as the 3xTF32
tensor-core work it issues (two passes over the upper-triangle tiles, 3 MMAs of 2 * 128 * 128 * d flop per tile) and set
beside a cuBLAS TF32 GEMM (torch.matmul with TF32 allowed) timed in the same run.  Prints the card's name and power limit
first, then one JSON line per measurement.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:            # noqa: BLE001
        return f"unknown ({e})"


def clustered(n, d, per, seed, noise):
    g = torch.Generator(device="cuda").manual_seed(seed)
    c = torch.randn(-(-n // per), d, device="cuda", generator=g)
    x = c.repeat_interleave(per, dim=0)[:n] + torch.randn(n, d, device="cuda", generator=g) * noise
    return x[torch.randperm(n, device="cuda", generator=g)].contiguous()


def timed(fn, reps):
    out, ms = None, []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return out, float(np.median(ms))


def cublas_tf32_tflops(d, reps=10):
    torch.backends.cuda.matmul.allow_tf32 = True
    a = torch.randn(16384, d, device="cuda")
    b = torch.randn(d, 16384, device="cuda")
    torch.matmul(a, b)
    _, ms = timed(lambda: torch.matmul(a, b), reps)
    torch.backends.cuda.matmul.allow_tf32 = False
    return 2.0 * 16384 * 16384 * d / (ms * 1e-3) / 1e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="20000x512,130000x2048")
    ap.add_argument("--degrees", default="10,300")
    ap.add_argument("--budget", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    from active_learning_b200.engine import Engine
    eng = Engine()
    print(json.dumps({"card": card()}), flush=True)
    for size in args.sizes.split(","):
        n, d = (int(v) for v in size.split("x"))
        gemm = cublas_tf32_tflops(d)
        nt = -(-n // 128)
        k13_flop = 2 * (nt * (nt + 1) // 2) * 3 * 2.0 * 128 * 128 * (-(-d // 32) * 32)
        for deg in (int(v) for v in args.degrees.split(",")):
            x = clustered(n, d, deg, n + deg, noise=0.35 / np.sqrt(d))
            eng.probcover_graph(x, 0.8)                       # warm-up: module load, scratch
            (row_ptr, cols, rech), g_ms = timed(lambda: eng.probcover_graph(x, 0.8), args.reps)
            lab = torch.zeros(n, dtype=torch.uint8, device="cuda")
            lab[torch.randperm(n, device="cuda")[:n // 100]] = 1
            budget = min(args.budget, n)
            eng.probcover_select(row_ptr, cols, lab, budget)
            (picks, steps), s_ms = timed(lambda: eng.probcover_select(row_ptr, cols, lab, budget), args.reps)
            print(json.dumps({"n": n, "d": d, "cluster": deg, "delta": 0.8, "nnz": int(cols.numel()),
                              "mean_degree": round(cols.numel() / n, 2), "recheck_pairs": rech,
                              "k13_ms": round(g_ms, 3), "k13_tflops_3xtf32": round(k13_flop / (g_ms * 1e-3) / 1e12, 1),
                              "cublas_tf32_tflops": round(gemm, 1), "budget": budget, "greedy_steps": steps,
                              "k14_ms": round(s_ms, 3)}), flush=True)
            del row_ptr, cols, x
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
