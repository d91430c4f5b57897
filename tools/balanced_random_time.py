"""BalancedRandomSampler's query on the H100: the reference's loop (tests/balanced_random_oracle.py, which keeps the
reference's per-class `torch.where(...).nonzero()` scans and its threshold loop) against the sampler (K10), the two arms
alternated in one run after a warm-up, with the sampler's parts timed separately.

    python tools/balanced_random_time.py [--n 1281167] [--classes 1000] [--eval 12000] [--budget 10000] [--rounds 3]

The pool is ImageNet-sized by default: labels drawn uniformly from the classes, held as a Python list like a dataset's
`targets`, `--eval` rows excluded.  Parts of the sampler: the targets list to an int32 array and its copy to the device,
K10 counts (CUDA events; the call synchronises once to check the labels) and the copy of C ints back, the host water-fill
plus the `torch.randperm` draws, K10 pick (CUDA events) and the copy of B ints back.  Both arms draw from the same torch
seed and must return the same list.  Prints one JSON line per measurement, the card's name and power limit first.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import balanced_random_oracle as BR  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:            # noqa: BLE001
        q = f"unknown ({e})"
    return q


class Pool(torch.utils.data.Dataset):
    def __init__(self, targets, num_classes):
        self.targets, self.num_classes = targets, num_classes

    def __len__(self):
        return len(self.targets)

    def __getitem__(self, i):
        return torch.tensor(float(i)), self.targets[i], i


def timed_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return out, a.elapsed_time(b)


def parts(s, budget):
    """The sampler's query split into its steps (same calls as BalancedRandomQuery.query), in ms."""
    from active_learning_b200.query_strategies.balanced_random import _host_labels, balanced_class_budgets
    eng, c = s.get_engine(), s.num_classes
    t = {}
    t0 = time.perf_counter()
    avail_h = np.ascontiguousarray(s.available_query_idxs(boolean=True), dtype=bool)
    budget = int(min(int(avail_h.sum()), budget))
    labels_h = _host_labels(s.al_set.targets)
    lab32 = np.clip(labels_h, -1, c).astype(np.int32)
    t["targets_to_array_ms"] = (time.perf_counter() - t0) * 1e3
    t0 = time.perf_counter()
    labels = torch.from_numpy(lab32).cuda()
    avail = torch.from_numpy(avail_h.view(np.uint8)).cuda()
    torch.cuda.synchronize()
    t["h2d_ms"] = (time.perf_counter() - t0) * 1e3
    counts_d, t["k10_counts_ms"] = timed_ms(lambda: eng.class_counts(labels, avail, c))
    t0 = time.perf_counter()
    counts = counts_d.cpu().numpy()
    t["d2h_counts_ms"] = (time.perf_counter() - t0) * 1e3
    t0 = time.perf_counter()
    k = balanced_class_budgets(counts, budget, c)
    perms = [torch.randperm(int(counts[cls]))[:int(k[cls])] for cls in np.flatnonzero(k > 0)]
    perm = torch.cat(perms)
    t["host_waterfill_randperm_ms"] = (time.perf_counter() - t0) * 1e3
    picks_d, t["k10_pick_ms"] = timed_ms(lambda: eng.class_pick(labels, avail, k, perm))   # includes the H2D of k, perm
    t0 = time.perf_counter()
    picks = picks_d.cpu().numpy().tolist()
    t["d2h_picks_ms"] = (time.perf_counter() - t0) * 1e3
    return picks, t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1281167)
    ap.add_argument("--classes", type=int, default=1000)
    ap.add_argument("--eval", type=int, default=12000)
    ap.add_argument("--budget", type=int, default=10000)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    from active_learning_b200.engine import Engine
    from active_learning_b200.query_strategies.get_strategy import get_strategy
    print(json.dumps({"card": card(), "torch_device": torch.cuda.get_device_name()}), flush=True)
    rng = np.random.default_rng(0)
    targets = rng.integers(0, a.classes, a.n).tolist()
    ev = rng.choice(a.n, a.eval, replace=False)
    ds = Pool(targets, a.classes)
    s = get_strategy("BalancedRandomSampler")(ds, ds, None, {"loader_te_args": {"batch_size": 256}}, ev, None, None,
                                              ckpt_path=tempfile.mkdtemp(prefix="alq_time_"), exp_name="t")
    s.set_engine(Engine())
    mask = s.available_query_idxs(boolean=True)
    budget = float(a.budget)
    torch.manual_seed(0)
    s.query(budget)                                               # warm-up: context, scratch, kernels
    parts(s, budget)
    ref_s, acc_s = [], []
    for r in range(a.rounds):
        torch.manual_seed(r)
        t0 = time.perf_counter()
        ref, _ = BR.balanced_random_query(targets, mask, a.classes, budget)
        ref_s.append(time.perf_counter() - t0)
        torch.manual_seed(r)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        got, _ = s.query(budget)
        acc_s.append(time.perf_counter() - t0)
        if got != ref:
            raise SystemExit(f"round {r}: the sampler's picks differ from the reference loop's")
        torch.manual_seed(r)
        picks, t = parts(s, budget)
        assert picks == got
        print(json.dumps({"round": r, "reference_loop_s": round(ref_s[-1], 4), "sampler_s": round(acc_s[-1], 4),
                          **{k: round(v, 3) for k, v in t.items()}}), flush=True)
    print(json.dumps({"n": a.n, "classes": a.classes, "eval": a.eval, "budget": a.budget,
                      "reference_loop_s": [round(x, 4) for x in ref_s], "sampler_s": [round(x, 4) for x in acc_s],
                      "speedup_median": round(float(np.median(ref_s) / np.median(acc_s)), 1), "same_picks": True}),
          flush=True)


if __name__ == "__main__":
    main()
