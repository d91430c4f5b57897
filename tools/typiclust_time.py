"""TypiClustSampler's kernels on the H100: the k-means++ seeding (K5's D^2 cold start), one K15 assignment and one K16
update, the Lloyd iteration count, K17 over one cycle of the walk, and the whole query on a synthetic pool, timed with
CUDA events after a warm-up.

    python tools/typiclust_time.py [--sizes 20000x512,130000x2048] [--ks 20,500] [--reps 3]

The rows are clustered (centres plus noise).  K15's rate is the 3xTF32 tensor-core work it issues (3 MMAs of
2 * 128 * 128 * d flop per row block x centre tile, d padded to 32) set beside a cuBLAS TF32 GEMM (torch.matmul with
TF32 allowed) timed in the same run; K17's work is counted in fp64 pair-columns (sum over the groups of m^2 d).  Prints
the card's name, power limit and max SM clock first, then one JSON line per shape.  The seeding is timed together with
the first assignment (kmeans with max_iter = 1).
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
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:            # noqa: BLE001
        return f"unknown ({e})"


def clustered(n, d, k, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    c = torch.randn(k, d, device="cuda", generator=g)
    return (c[torch.randint(0, k, (n,), device="cuda", generator=g)]
            + 0.6 * torch.randn(n, d, device="cuda", generator=g)).contiguous()


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


def query_time(eng, x, k, reps):
    """The whole query (pool forward excluded: the embeddings are given) on a pool with no labeled row and budget k."""
    from helpers import make_strategy
    n = x.shape[0]
    s = make_strategy("TypiClustSampler", torch.zeros(n, 4), x.cpu(), [], [], 1024, engine=eng)
    s._features = lambda idxs: (x[torch.as_tensor(idxs, device=x.device)], None)
    np.random.seed(0)
    s.query(k)
    return timed(lambda: s.query(k), reps)[1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="20000x512,130000x2048")
    ap.add_argument("--ks", default="20,500")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    from active_learning_b200.engine import Engine
    from active_learning_b200.query_strategies.typiclust import cluster_order
    eng = Engine()
    print(json.dumps({"card": card()}), flush=True)
    for size in args.sizes.split(","):
        n, d = (int(v) for v in size.split("x"))
        gemm = cublas_tf32_tflops(d)
        x = clustered(n, d, 300, n + d)
        xhat = eng.normalize(x)
        rows = eng._kmeans_rows(xhat, False)
        for k in (int(v) for v in args.ks.split(",")):
            rng = np.random.default_rng(k)
            first, unif = int(rng.integers(n)), rng.random(k - 1)
            eng.kmeans(xhat, first, unif, k, max_iter=1)                      # warm-up: modules, scratch
            (_, centres, _, _), seed_ms = timed(lambda: eng.kmeans(xhat, first, unif, k, max_iter=1), args.reps)
            labels, centres, iters, _ = eng.kmeans(xhat, first, unif, k)
            lab = labels.clone()
            (_, rech), a_ms = timed(lambda: eng._assign(rows, centres, lab), args.reps)
            c2 = centres.clone()
            _, u_ms = timed(lambda: eng.kmeans_update(xhat, labels, c2), args.reps)
            lab_h = labels.cpu().numpy().astype(np.int64)
            order = cluster_order(lab_h, np.zeros(n, dtype=bool), k, 5)
            groups = [np.flatnonzero(lab_h == c) for c in order]
            goff = np.concatenate([[0], np.cumsum([len(g) for g in groups])])
            flat = torch.from_numpy(np.concatenate(groups).astype(np.int32)).cuda()
            eng.typicality(xhat, flat, goff, 20)
            _, t_ms = timed(lambda: eng.typicality(xhat, flat, goff, 20), args.reps)
            q_ms = query_time(eng, x, k, args.reps)
            dp = -(-d // 32) * 32
            k15_flop = -(-n // 128) * -(-k // 128) * 3 * 2.0 * 128 * 128 * dp
            pair_cols = float(sum(len(g) ** 2 for g in groups)) * d
            print(json.dumps({"n": n, "d": d, "K": k, "seeding_and_first_assign_ms": round(seed_ms, 3),
                              "lloyd_assignments": iters,
                              "k15_ms": round(a_ms, 3), "k15_rechecked_rows": rech,
                              "k15_tflops_3xtf32": round(k15_flop / (a_ms * 1e-3) / 1e12, 1),
                              "cublas_tf32_tflops": round(gemm, 1), "k16_ms": round(u_ms, 3),
                              "k17_groups": len(groups), "k17_ms": round(t_ms, 3),
                              "k17_pair_columns": pair_cols, "query_budget": k, "query_ms": round(q_ms, 3)}), flush=True)
        del x, xhat, rows
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
