"""CALSampler's kernels on the H100: K18 (the exact k nearest labeled rows), K19 (the contrastive scores) and the whole
query with the embeddings and logits given, timed with CUDA events (the median of --reps after a warm-up).

    python tools/cal_time.py [--sizes 20000x512:5000,130000x2048:50000] [--classes 10,1000] [--reps 3]

A size NxD:M is a pool of N rows of width D whose first M rows are labeled (the references) and the rest the candidates,
clustered (300 centres plus noise).  k = 10.  K18's rate is the 3xTF32 tensor-core work it issues (3 MMAs of
2 * 128 * 128 * d flop per row block x column tile, d padded to 32) set beside a cuBLAS TF32 GEMM (torch.matmul with TF32
allowed) timed in the same run; its fallback count is the rows the screen could not certify.  The query's budget is a
fifth of the candidates.  Prints the card's name, power limit and max SM clock first, then one JSON line per shape.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from typiclust_time import card, clustered, cublas_tf32_tflops, timed  # noqa: E402

K = 10


def query_time(eng, emb, logits, n_lab, budget, reps):
    """The whole query (pool forward excluded: the embeddings and logits are given)."""
    from helpers import make_strategy
    n = emb.shape[0]
    s = make_strategy("CALSampler", torch.zeros(n, 1), torch.zeros(n, 4), [], np.arange(n_lab), 1024, engine=eng)

    def forward(idxs, net, want_features):
        t = torch.as_tensor(idxs, device=emb.device)
        return logits[t], emb[t]
    s._forward_pool = forward
    np.random.seed(0)
    s.query(budget)
    return timed(lambda: s.query(budget), reps)[1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="20000x512:5000,130000x2048:50000")
    ap.add_argument("--classes", default="10,1000")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    from active_learning_b200.engine import Engine
    eng = Engine()
    print(json.dumps({"card": card()}), flush=True)
    for size in args.sizes.split(","):
        shape, m = size.split(":")
        n, d = (int(v) for v in shape.split("x"))
        m = int(m)
        gemm = cublas_tf32_tflops(d)
        emb = clustered(n, d, 300, n + d)
        y, x = emb[:m], emb[m:]
        eng.knn(x, y, K)                                                       # warm-up: modules, scratch
        (idx, _, fb), k18_ms = timed(lambda: eng.knn(x, y, K), args.reps)
        dp = -(-d // 32) * 32
        k18_flop = -(-x.shape[0] // 128) * -(-m // 128) * 3 * 2.0 * 128 * 128 * dp
        for c in (int(v) for v in args.classes.split(",")):
            g = torch.Generator(device="cuda").manual_seed(c)
            logits = torch.randn(n, c, device="cuda", generator=g) * 3
            zc, zr = logits[m:].contiguous(), logits[:m].contiguous()
            eng.cal_scores(zc, zr, idx)
            _, k19_ms = timed(lambda: eng.cal_scores(zc, zr, idx), args.reps)
            budget = x.shape[0] // 5
            q_ms = query_time(eng, emb, logits, m, budget, args.reps)
            print(json.dumps({"n_candidates": x.shape[0], "m_labeled": m, "d": d, "C": c, "k": K,
                              "k18_ms": round(k18_ms, 3), "k18_fallback_rows": fb,
                              "k18_tflops_3xtf32": round(k18_flop / (k18_ms * 1e-3) / 1e12, 1),
                              "cublas_tf32_tflops": round(gemm, 1), "k19_ms": round(k19_ms, 3),
                              "query_budget": budget, "query_ms": round(q_ms, 3)}), flush=True)
            del logits, zc, zr
        del emb, x, y, idx
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
