"""MaxHerdingSampler on the H100: K22 (the Gaussian kernel matrix), K23's set-up and its greedy loop, and the whole query,
timed with CUDA events after a warm-up, with the rows the picks changed (sum of |S_t|) and the launch count.  At CIFAR-10's
shape a plain torch loop (the full-matrix gain at every step) runs on the same matrix and its picks are compared.

    python tools/maxherding_time.py [--shapes NxD:L:B,...] [--sigma S] [--reps R] [--torch-loop-max N]

A shape NxD:L:B is n rows of width d, L labeled rows (a fraction < 1 is a share of n) and budget B.  The rows are
clustered (centres plus noise; see `clustered`), normalised by the engine.  Prints the card, its power limit and max SM
clock first, then one JSON line per shape.
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


def clustered(n, d, per, seed, noise):
    g = torch.Generator(device="cuda").manual_seed(seed)
    c = torch.randn(-(-n // per), d, device="cuda", generator=g)
    x = c[torch.randint(0, c.shape[0], (n,), device="cuda", generator=g)]
    return x + noise * torch.randn(n, d, device="cuda", generator=g)


def timed(fn, reps):
    ms = []
    for _ in range(reps):
        out = None                                                     # the previous result is freed first
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return out, float(np.median(ms))


def torch_loop(K, lab, avail, budget):
    """The obvious loop: every step recomputes every gain from the whole matrix (fp32 sums)."""
    n = K.shape[0]
    idx = torch.nonzero(lab).flatten()
    m = K[idx].max(dim=0).values if idx.numel() else torch.zeros(n, device=K.device)
    cand = avail.clone().bool()
    picks = []
    for _ in range(budget):
        gain = torch.zeros(n, device=K.device)
        for lo in range(0, n, 8192):
            gain += (K[lo:lo + 8192] - m[lo:lo + 8192, None]).clamp_min_(0).sum(dim=0)
        c = int(torch.where(cand, gain, torch.tensor(-1.0, device=K.device)).argmax())
        picks.append(c)
        m = torch.maximum(m, K[c])
        cand[c] = False
    return np.asarray(picks)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="50000x512:0:100,50000x512:0:1000,50000x512:1000:100,50000x512:1000:1000,"
                                        "115846x2048:0.1:10000")
    ap.add_argument("--sigma", type=float, default=0.5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--torch-loop-max", type=int, default=50000, help="run the torch loop up to this n")
    args = ap.parse_args()
    from active_learning_b200.engine import Engine
    from helpers import make_strategy
    eng = Engine()
    print(json.dumps({"card": card()}), flush=True)
    for shape in args.shapes.split(","):
        nd, nl, b = shape.split(":")
        n, d = (int(v) for v in nd.split("x"))
        n_lab = int(float(nl) * n) if float(nl) < 1 else int(nl)
        budget = int(b)
        x = clustered(n, d, 20, n + d, noise=0.3)
        xhat = eng.normalize(x)
        eng.herding_kernel(xhat, args.sigma)                          # warm-up
        torch.cuda.empty_cache()
        K, k22_ms = timed(lambda: eng.herding_kernel(xhat, args.sigma), args.reps)
        rng = np.random.default_rng(1)
        lab_np = np.zeros(n, dtype=bool)
        lab_np[rng.choice(n, n_lab, replace=False)] = True
        lab = torch.from_numpy(lab_np).cuda()
        avail = ~lab
        eng.herding_select(K, lab, avail, min(budget, 10))             # warm-up
        _, setup_ms = timed(lambda: eng.herding_select(K, lab, avail, 0), args.reps)
        l0 = eng.launches
        (picks, m, sum_s), sel_ms = timed(lambda: eng.herding_select(K, lab, avail, budget), args.reps)
        launches = (eng.launches - l0) // args.reps
        rec = {"n": n, "d": d, "labeled": n_lab, "budget": budget, "sigma": args.sigma,
               "k22_ms": round(k22_ms, 2), "k23_setup_ms": round(setup_ms, 2), "k23_loop_ms": round(sel_ms - setup_ms, 2),
               "k23_ms": round(sel_ms, 2), "sum_S": sum_s, "mean_S": round(sum_s / max(len(picks), 1), 1),
               "k23_launches": launches, "loop_us_per_step": round(1e3 * (sel_ms - setup_ms) / max(len(picks), 1), 2)}
        if n <= args.torch_loop_max:
            tp, t_ms = timed(lambda: torch_loop(K, lab, avail, budget), 1)
            rec.update({"torch_loop_ms": round(t_ms, 1), "torch_loop_same_order": float(np.mean(tp == picks)),
                        "torch_loop_same_set": len(set(tp.tolist()) & set(picks.tolist())) / len(picks)})
        del K, m
        torch.cuda.empty_cache()
        # the whole query: embeddings given, through the sampler (pool shuffles, normalise, K22, K23, release)
        emb = x.cpu()
        del x, xhat
        torch.cuda.empty_cache()
        s = make_strategy("MaxHerdingSampler", torch.zeros(n, 4), emb, np.arange(0), np.flatnonzero(lab_np), 4096,
                          engine=eng, sigma=args.sigma)
        np.random.seed(0)
        _, q_ms = timed(lambda: s.query(budget), 1)
        rec["query_ms"] = round(q_ms, 1)
        print(json.dumps(rec), flush=True)
        del s, emb
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
