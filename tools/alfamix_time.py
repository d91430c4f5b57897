"""ALFAMixSampler's kernels on the H100: K20 (the closed-form mixing test per row), K21 (each cluster's row nearest its
centre) and the whole query with the embeddings and logits given, timed with CUDA events (the median of --reps after a
warm-up).

    python tools/alfamix_time.py [--shapes 50000x512:10:1000,115846x2048:1000:10000] [--reps 3]

A shape NxD:C:B is a pool of N clustered rows (300 centres plus noise) of width D, a random head of C classes, 10 % of
the rows labeled with random classes, and the budget B.  K20 runs on the candidates (the unlabeled rows); K21 on the
L2-normalised candidates with K = B clusters and the labels of one K15 assignment against B of them.  The query's time
is split into K20, the k-means (seeding and Lloyd) and the rest.  Prints the card's name, power limit and max SM clock
first, then one JSON line per shape.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from typiclust_time import card, clustered, timed  # noqa: E402


def query_time(eng, emb, logits, weight, ys, n_lab, budget, reps):
    """The whole query (pool forward excluded: the embeddings and logits are given), with the time inside K20 and inside
    the k-means of the last run."""
    from helpers import HeadNet, LabeledIndexDataset, make_strategy
    n, c = logits.shape
    net = HeadNet(torch.zeros(n, 1), weight.cpu(), torch.zeros(c))
    s = make_strategy("ALFAMixSampler", None, None, [], np.arange(n_lab), 1024, engine=eng, net=net,
                      dataset=LabeledIndexDataset(ys, c))
    s.net.cuda()

    def forward(idxs, net, want_features):
        t = torch.as_tensor(idxs, device=emb.device)
        return logits[t], emb[t]
    s._forward_pool = forward
    spent = {}

    def clocked(name, fn):
        def run(*a, **k):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fn(*a, **k)
            torch.cuda.synchronize()
            spent[name] = spent.get(name, 0.0) + (time.perf_counter() - t0) * 1e3
            return out
        return run
    np.random.seed(0)
    s.query(budget)
    q_ms = timed(lambda: (np.random.seed(0), s.query(budget)), reps)[1]
    rho_fn, km_fn = eng.alfamix_rho, eng.kmeans
    eng.alfamix_rho, eng.kmeans = clocked("k20", rho_fn), clocked("kmeans", km_fn)
    try:
        np.random.seed(0)
        s.query(budget)
    finally:
        eng.alfamix_rho, eng.kmeans = rho_fn, km_fn
    return q_ms, spent


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="50000x512:10:1000,115846x2048:1000:10000")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    from active_learning_b200.engine import Engine
    eng = Engine()
    print(json.dumps({"card": card()}), flush=True)
    for shape in args.shapes.split(","):
        nd, c, budget = shape.split(":")
        n, d = (int(v) for v in nd.split("x"))
        c, budget = int(c), int(budget)
        m = n // 10
        emb = clustered(n, d, 300, n + d)
        g = torch.Generator(device="cuda").manual_seed(c)
        weight = torch.randn(c, d, device="cuda", generator=g) * 0.05
        logits = emb @ weight.T
        ys = np.random.default_rng(c).integers(0, c, size=n)
        x, z = emb[m:], logits[m:]
        anc = emb[:c].contiguous()
        eng.alfamix_rho(z, x, anc, weight)                                     # warm-up: modules, scratch
        _, k20_ms = timed(lambda: eng.alfamix_rho(z, x, anc, weight), args.reps)
        xhat = eng.normalize(x)
        cen = xhat[torch.randperm(x.shape[0], device="cuda", generator=g)[:budget]].contiguous()
        labels, _, _ = eng.kmeans_assign(xhat, cen)
        eng.kmeans_nearest(xhat, labels, cen)
        _, k21_ms = timed(lambda: eng.kmeans_nearest(xhat, labels, cen), args.reps)
        q_ms, spent = query_time(eng, emb, logits, weight, ys, m, budget, args.reps)
        print(json.dumps({"n_candidates": x.shape[0], "d": d, "C": c, "budget": budget,
                          "k20_ms": round(k20_ms, 3), "k21_ms": round(k21_ms, 3), "query_ms": round(q_ms, 3),
                          "query_k20_ms": round(spent.get("k20", 0.0), 3),
                          "query_kmeans_ms": round(spent.get("kmeans", 0.0), 3)}), flush=True)
        del emb, logits, x, z, xhat, cen, labels
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
