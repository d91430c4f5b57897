"""BalancingSampler at ImageNet-LT's 1 000 classes on the H100: K12 (the persistent loop over the incremental row x
class table) against the per-step path, alternated after a warm-up.

    python tools/balancing_table_time.py [--rounds 3]

Shapes:
  lt     ImageNet-LT: 115 846 rows x 2048 with the class sizes of ImageNet_LT_train.txt (the `lt_counts` fixture of
         tests/golden/reference_golden_balancing_table.npz), a tenth labeled; K12 at budgets 1 000 and 10 000 and the
         per-step path (option balancing_loop = 1, through the sampler) at 1 000;
  cifar  20 431 rows x 512, C = 1000, 1 000 labeled rows with an exp imbalance of 0.1, budget 100: K12 and the per-step
         path.
Per round and arm: the wall time of the query (ended by a device synchronise) and the balancing steps.  The time per
balancing step is the difference between K12's two budgets over the difference of their balancing steps (the set-up
and the table build cancel), and the floor n_avail * (4 d + 8 C + 9) bytes per step over it is given as a share of the
H100 SXM data sheet's 3.35 TB/s HBM bound.  The picks of the two paths at the same budget and seed are compared.
Prints one JSON line per measurement, the card's name, power limit and maximum SM clock first.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
HBM = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:            # noqa: BLE001
        q = f"unknown ({e})"
    return q


def pool(ys, d, n_lab, seed):
    n, c = len(ys), int(ys.max()) + 1
    g = torch.Generator(device="cuda").manual_seed(seed)
    yt = torch.from_numpy(ys).cuda()
    centres = torch.randn(c, d, device="cuda", generator=g)
    emb = torch.relu(centres[yt] * 0.5 + torch.randn(n, d, device="cuda", generator=g))
    lab = np.sort(np.random.default_rng(seed).choice(n, size=n_lab, replace=False))
    return emb.contiguous(), lab


def k12(eng, emb, ys, lab, c, budget, seed):
    """-> (picks, seconds, balancing steps) of one direct K12 query under auto."""
    n = emb.shape[0]
    avail = np.ones(n, dtype=np.uint8)
    avail[lab] = 0
    labels = torch.from_numpy(ys.astype(np.int32)).cuda()
    av, lb = torch.from_numpy(avail).cuda(), torch.from_numpy(1 - avail).cuda()
    xn = eng.row_norm2(emb)
    np.random.seed(seed)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    assert eng.balancing_select(emb, xn, labels, av, lb, c, budget) is None      # K11 declines at this C
    got = eng.balancing_table_select(emb, xn, labels, av, lb, c, budget)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    assert got is not None, "K12 declined"
    return [int(i) for i in got[0]], dt, got[1]


def per_step(eng, emb, ys, lab, c, budget, seed):
    from helpers import LabeledIndexDataset, make_strategy
    s = make_strategy("BalancingSampler", torch.zeros(emb.shape[0], c, device=emb.device), emb,
                      np.zeros(0, dtype=np.int64), lab, 4096, engine=eng, dataset=LabeledIndexDataset(ys, c))
    eng.set_option("balancing_loop", 1)
    try:
        np.random.seed(seed)
        torch.cuda.synchronize()
        l0, t0 = eng.launches, time.perf_counter()
        idx, _ = s.query(float(budget))
        torch.cuda.synchronize()
        return [int(i) for i in idx], time.perf_counter() - t0, eng.launches - l0
    finally:
        eng.set_option("balancing_loop", 0)


def same(a, b):
    return int(sum(x == y for x, y in zip(a, b)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    from active_learning_b200.engine import Engine
    print(json.dumps({"card": card(), "torch_device": torch.cuda.get_device_name()}), flush=True)
    eng = Engine()
    counts = np.load(os.path.join(ROOT, "tests", "golden", "reference_golden_balancing_table.npz"))["lt_counts"]

    # ---- ImageNet-LT ----
    c, d = 1000, 2048
    ys = np.random.default_rng(3).permutation(np.repeat(np.arange(c), counts))
    n = len(ys)
    emb, lab = pool(ys, d, n // 10, 7)
    n_avail = n - len(lab)
    floor_s = n_avail * (4 * d + 8 * c + 9) / HBM
    k12(eng, emb, ys, lab, c, 50, 1)                         # warm-up: context, scratch, kernels
    per_step(eng, emb, ys, lab, c, 5, 1)
    rows = []
    for r in range(a.rounds):
        p1, t1, b1 = k12(eng, emb, ys, lab, c, 1000, 100 + r)
        ps, ts, ls = per_step(eng, emb, ys, lab, c, 1000, 100 + r)
        p2, t2, b2 = k12(eng, emb, ys, lab, c, 10000, 100 + r)
        step = (t2 - t1) / max(b2 - b1, 1)
        rows.append((t1, t2, ts, step))
        print(json.dumps({"shape": "lt", "round": r, "k12_1000_s": round(t1, 4), "k12_1000_balancing_steps": b1,
                          "k12_10000_s": round(t2, 4), "k12_10000_balancing_steps": b2,
                          "per_step_1000_s": round(ts, 4), "per_step_launches": ls,
                          "k12_ms_per_balancing_step": round(1e3 * step, 4),
                          "floor_share_of_hbm_bound": round(floor_s / step, 3),
                          "same_picks_1000": same(p1, ps), "same_prefix_10000": same(p1, p2[:1000])}), flush=True)
    med = np.median(np.array(rows), axis=0)
    print(json.dumps({"shape": "lt", "n": n, "d": d, "classes": c, "labeled": int(len(lab)), "n_avail": n_avail,
                      "median_k12_1000_s": round(med[0], 4), "median_k12_10000_s": round(med[1], 4),
                      "median_per_step_1000_s": round(med[2], 4), "median_k12_ms_per_balancing_step": round(1e3 * med[3], 4),
                      "floor_ms_per_step": round(1e3 * floor_s, 4), "floor_share_of_hbm_bound": round(floor_s / med[3], 3)}),
          flush=True)
    del emb
    torch.cuda.empty_cache()

    # ---- CIFAR-10-LT's shape at C = 1000 ----
    c, d, n, budget = 1000, 512, 20431, 100
    ys = np.random.default_rng(5).integers(0, c, size=n)
    emb, _ = pool(ys, d, 1, 9)
    want = [max(1, int(1000 * 0.1 ** (k / (c - 1)) / sum(0.1 ** (j / (c - 1)) for j in range(c)))) for k in range(c)]
    rng = np.random.default_rng(9)
    lab = np.sort(np.concatenate([rng.choice(np.flatnonzero(ys == k), size=min(want[k], int((ys == k).sum())), replace=False)
                                  for k in range(c) if (ys == k).any()]))
    k12(eng, emb, ys, lab, c, 10, 1)
    per_step(eng, emb, ys, lab, c, 10, 1)
    for r in range(a.rounds):
        p1, t1, b1 = k12(eng, emb, ys, lab, c, budget, 200 + r)
        ps, ts, ls = per_step(eng, emb, ys, lab, c, budget, 200 + r)
        print(json.dumps({"shape": "cifar_c1000", "round": r, "n": n, "d": d, "budget": budget, "k12_s": round(t1, 4),
                          "k12_balancing_steps": b1, "per_step_s": round(ts, 4), "per_step_launches": ls,
                          "same_picks": same(p1, ps)}), flush=True)


if __name__ == "__main__":
    main()
