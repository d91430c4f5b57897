"""BalancingSampler's query on the H100: the per-step path (one K3 pair, one ratio arg-min and two host round trips per
pick) against K11, the persistent loop, through the sampler itself, the arms alternated after a warm-up.

    python tools/balancing_time.py [--rounds 3] [--skip-big] [--skip-host]

Shapes:
  cifar   CIFAR-10-LT: 20 431 rows x 512 (SSLResNet18), C = 10, 1 000 labeled rows with an exp imbalance of factor 0.1,
          budget 1 000; also the oracle's loop on the host (oracle/al_oracle.py balancing_query, torch on the CPU),
          timed once;
  big     200 000 rows x 2048, C = 10, 2 000 labeled rows (same imbalance), budget 10 000;
  beyond  C = 1000 at 20 431 x 512, budget 100: beyond the loop's shared-memory limit, so auto runs the per-step path.
Each query starts from the same NumPy seed; the picks of the arms are compared (they agree wherever the two best ratios
of every balancing step are further apart than fp32 rounding).  The embeddings stay cached on the device across the
queries (freeze_feature), so the pool forward is not timed.  Prints one JSON line per measurement, the card's name and
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:            # noqa: BLE001
        q = f"unknown ({e})"
    return q


def pool(n, d, c, n_lab, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    ys = torch.randint(0, c, (n,), device="cuda", generator=g)
    centres = torch.randn(c, d, device="cuda", generator=g) * 2
    emb = torch.relu(centres[ys] + torch.randn(n, d, device="cuda", generator=g))
    ys = ys.cpu().numpy()
    want = [max(1, int(n_lab * 0.1 ** (k / max(c - 1, 1)) / sum(0.1 ** (j / max(c - 1, 1)) for j in range(c))))
            for k in range(c)]
    rng = np.random.default_rng(seed)
    lab = np.concatenate([rng.choice(np.flatnonzero(ys == k), size=min(want[k], int((ys == k).sum())), replace=False)
                          for k in range(c)])
    return emb, ys, np.sort(lab)


def strategy(emb, ys, lab, c, eng):
    from helpers import LabeledIndexDataset, make_strategy
    return make_strategy("BalancingSampler", torch.zeros(emb.shape[0], c, device=emb.device), emb,
                         np.zeros(0, dtype=np.int64), lab, 4096, engine=eng, dataset=LabeledIndexDataset(ys, c))


def query(s, eng, loop, budget, seed):
    """-> (picks, seconds, launches) of one query with option balancing_loop = loop (1 per-step, 2 persistent, 0 auto)."""
    eng.set_option("balancing_loop", loop)
    np.random.seed(seed)
    torch.cuda.synchronize()
    l0, t0 = eng.launches, time.perf_counter()
    idx, _ = s.query(float(budget))
    torch.cuda.synchronize()
    dt, dl = time.perf_counter() - t0, eng.launches - l0
    eng.set_option("balancing_loop", 0)
    return [int(i) for i in idx], dt, dl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--skip-big", action="store_true")
    ap.add_argument("--skip-host", action="store_true")
    a = ap.parse_args()
    from active_learning_b200.engine import Engine
    print(json.dumps({"card": card(), "torch_device": torch.cuda.get_device_name()}), flush=True)
    eng = Engine()
    shapes = [("cifar", 20431, 512, 10, 1000, 1000, a.rounds, True)]
    if not a.skip_big:
        shapes.append(("big", 200000, 2048, 10, 2000, 10000, 1, True))
    shapes.append(("beyond", 20431, 512, 1000, 1000, 100, 1, False))
    for name, n, d, c, n_lab, budget, rounds, loop_fits in shapes:
        emb, ys, lab = pool(n, d, c, n_lab, 7)
        s = strategy(emb, ys, lab, c, eng)
        rec = {"shape": name, "n": n, "d": d, "classes": c, "labeled": int(len(lab)), "budget": budget}
        if loop_fits:
            query(s, eng, 2, min(budget, 50), 1)                 # warm-up: forward pass cached, context, kernels
            query(s, eng, 1, 20, 1)
            step_s, loop_s, same = [], [], []
            for r in range(rounds):
                p1, t1, l1 = query(s, eng, 1, budget, 100 + r)
                p2, t2, l2 = query(s, eng, 2, budget, 100 + r)
                step_s.append(t1)
                loop_s.append(t2)
                same.append(int(sum(x == y for x, y in zip(p1, p2))))
                rec.update(per_step_launches=l1, loop_launches=l2)
                print(json.dumps({"shape": name, "round": r, "per_step_s": round(t1, 4), "loop_s": round(t2, 4),
                                  "same_picks": same[-1], "of": len(p1)}), flush=True)
            rec.update(per_step_s=[round(x, 4) for x in step_s], loop_s=[round(x, 4) for x in loop_s],
                       per_step_ms_per_pick=round(1e3 * float(np.median(step_s)) / budget, 4),
                       loop_ms_per_pick=round(1e3 * float(np.median(loop_s)) / budget, 4),
                       speedup_median=round(float(np.median(step_s) / np.median(loop_s)), 2), same_picks=same)
            if name == "cifar" and not a.skip_host:
                from oracle import al_oracle as O
                lb = np.zeros(n, dtype=bool)
                lb[lab] = True
                np.random.seed(100)
                diag = {}
                t0 = time.perf_counter()
                ref, _ = O.balancing_query(emb.cpu(), torch.from_numpy(ys), ~lb, lb, budget, c, diag)
                rec.update(host_oracle_s=round(time.perf_counter() - t0, 3), host_balancing_steps=diag["balancing_steps"],
                           host_min_rel_gap=diag["min_rel_gap"])
                p2, _, _ = query(s, eng, 2, budget, 100)
                rec["host_same_picks"] = int(sum(x == y for x, y in zip(ref, p2)))
        else:
            x = emb.contiguous()
            declined = eng.balancing_select(x, eng.row_norm2(x), torch.from_numpy(ys.astype(np.int32)).cuda(),
                                            torch.ones(n, dtype=torch.uint8, device="cuda"),
                                            torch.zeros(n, dtype=torch.uint8, device="cuda"), c, budget) is None
            query(s, eng, 0, 10, 1)
            _, t, l = query(s, eng, 0, budget, 100)
            rec.update(loop_declined=declined, auto_s=round(t, 4), auto_launches=l)
        print(json.dumps(rec), flush=True)
        del s, emb
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
