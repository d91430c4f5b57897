"""K8 over the banded layout (alq_ward_nn_chain_banded) against K8 over the condensed vector, timed on one H100 with CUDA
events.

    python tools/ward_banded_time.py [--n 20000 80000] [--d 2048] [--repeats 3] [--out FILE]

For each n (post-ReLU Gaussian rows of width d), K7 writes scipy's condensed vector once; every timed K8 call consumes a
fresh copy of it.  Each repetition times, in an order that rotates from one repetition to the next, the condensed walk
and the banded walk over 1, 2, 4 and 8 bands of ward_bands(n, G) -- slices of one local vector, so only the band lookup
differs from the condensed walk.  The merge lists of every call must be identical (the tool exits non-zero otherwise).
Reports min / median / max per variant and the banded walk's median over the condensed one.  Prints the card's name and
power limit first, then one JSON line per measurement.  The distributed placement across several GPUs (peer reads
over NVLink) is not measured by this tool.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:    # noqa: BLE001
        return f"unknown ({e})"


def stats(ms):
    ms = sorted(ms)
    return {"min_ms": round(ms[0], 1), "median_ms": round(ms[len(ms) // 2], 1), "max_ms": round(ms[-1], 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[20000, 80000])
    ap.add_argument("--d", type=int, default=2048)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from active_learning_b200 import sharding
    from active_learning_b200.engine import Engine
    eng = Engine()
    results = [{"card": card(), "torch_device": torch.cuda.get_device_name(), "d": args.d,
                "gpus": torch.cuda.device_count(), "distributed_across_gpus": "not measured"}]
    print(json.dumps(results[0]), flush=True)

    def emit(rec):
        results.append(rec)
        print(json.dumps(rec), flush=True)

    ok = True
    for n in args.n:
        g = torch.Generator(device="cuda").manual_seed(n)
        x = torch.relu(torch.randn(n, args.d, device="cuda", generator=g))
        pristine = eng.pdist(x, condensed=True)
        del x
        work = torch.empty_like(pristine)
        variants = ["condensed"] + [f"banded G={G}" for G in (1, 2, 4, 8)]
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

        def run(v):
            work.copy_(pristine)
            torch.cuda.synchronize()
            a.record()
            if v == "condensed":
                xy, md = eng.nn_chain(work, n)
            else:
                cuts = sharding.ward_bands(n, int(v.split("=")[1]))
                parts = [work[sharding.band_pairs(n, 0, lo):sharding.band_pairs(n, 0, hi)] if hi > lo else None
                         for lo, hi in zip(cuts, cuts[1:])]
                xy, md = eng.nn_chain_banded(cuts, parts, n)
            b.record()
            torch.cuda.synchronize()
            return a.elapsed_time(b), xy.cpu().numpy(), md.cpu().numpy().view(np.int64)

        eng.nn_chain(pristine[:1].clone(), 2)                             # warm-up: module load, first launches
        eng.nn_chain_banded([0, 2], [pristine[:1].clone()], 2)
        times = {v: [] for v in variants}
        ref = None
        for rep in range(args.repeats):
            order = variants[rep % len(variants):] + variants[:rep % len(variants)]
            for v in order:
                ms, xy, md = run(v)
                times[v].append(ms)
                if ref is None:
                    ref = (xy, md)
                elif not (np.array_equal(xy, ref[0]) and np.array_equal(md, ref[1])):
                    ok = False
                    emit({"n": n, "variant": v, "error": "merge list differs from the first call's"})
        base = sorted(times["condensed"])[len(times["condensed"]) // 2]
        for v in variants:
            med = sorted(times[v])[len(times[v]) // 2]
            emit({"n": n, "variant": v, **stats(times[v]), "median_over_condensed": round(med / base, 4),
                  "per_merge_us": round(1e3 * med / (n - 1), 2)})
        emit({"n": n, "merge_lists_identical": ok})
        del pristine, work
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
