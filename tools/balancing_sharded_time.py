"""BalancingSampler's K11 / K12 with rows sharded over G GPUs (one process per GPU, NCCL, Engine(rank).comm_init()).

    python tools/balancing_sharded_time.py [--rounds 3]

For every G from 1 to the device count, every rank builds the same replicated pool (seeded on the device) and runs:
  lt     ImageNet-LT: 115 846 rows x 2048 with the class sizes of ImageNet_LT_train.txt (the `lt_counts` fixture of
         tests/golden/reference_golden_balancing_table.npz), a tenth labeled, C = 1000: K12 at budgets 1 000 and 10 000;
  cifar  CIFAR-10-LT's shape: 20 431 rows x 512, C = 10, 1 000 labeled rows with an exp imbalance of 0.1: K11 at 1 000.
Each query is timed on rank 0 from a barrier to the end of the call (the call synchronises its stream).  The time per
balancing step is the difference between K12's two budgets over the difference of their balancing steps (the set-up
and the table build cancel).  Rank 0 also runs the unsharded single-GPU call on the same inputs, alternated with the
sharded one, and reports whether the picks, balancing steps and MT19937 state are the same on every rank and equal to
it.  At G = 1 the sharded call runs in a group of one rank, so the difference to the unsharded call is what the window
path costs.  A G larger than the device count is reported as "not measured".  Prints one JSON line per measurement,
the card's name, power limit and maximum SM clock first.
"""
import argparse
import json
import os
import socket
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:            # noqa: BLE001
        q = f"unknown ({e})"
    return q


def pool(ys, d, lab_rows, seed):
    """Replicated inputs: the same on every rank (device generator seeded alike)."""
    n, c = len(ys), int(ys.max()) + 1
    g = torch.Generator(device="cuda").manual_seed(seed)
    yt = torch.from_numpy(ys).cuda()
    centres = torch.randn(c, d, device="cuda", generator=g)
    emb = torch.relu(centres[yt] * 0.5 + torch.randn(n, d, device="cuda", generator=g)).contiguous()
    avail = np.ones(n, dtype=np.uint8)
    avail[lab_rows] = 0
    return emb, yt.to(torch.int32), torch.from_numpy(avail).cuda(), torch.from_numpy(1 - avail).cuda()


def shapes():
    counts = np.load(os.path.join(ROOT, "tests", "golden", "reference_golden_balancing_table.npz"))["lt_counts"]
    ys = np.random.default_rng(3).permutation(np.repeat(np.arange(1000), counts))
    lt_lab = np.sort(np.random.default_rng(7).choice(len(ys), size=len(ys) // 10, replace=False))
    c, n = 10, 20431
    ys10 = np.random.default_rng(5).integers(0, c, size=n)
    want = [int(1000 * 0.1 ** (k / (c - 1)) / sum(0.1 ** (j / (c - 1)) for j in range(c))) for k in range(c)]
    rng = np.random.default_rng(9)
    cifar_lab = np.sort(np.concatenate([rng.choice(np.flatnonzero(ys10 == k), size=want[k], replace=False)
                                        for k in range(c)]))
    return {"lt": (ys, 2048, lt_lab, 1000, (1000, 10000), "balancing_table_select"),
            "cifar": (ys10, 512, cifar_lab, c, (1000,), "balancing_select")}


def _worker(rank, world, port, rounds, out_path):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    import torch.distributed as dist
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from active_learning_b200.engine import Engine
    from active_learning_b200.sharding import ShardGroup
    eng = Engine(rank).comm_init()
    group = ShardGroup()
    out = []

    def call(fn, args, budget, seed, shard_off):
        if shard_off is not None:                                         # collective; an unsharded call is rank 0's alone
            dist.barrier()
        np.random.seed(seed)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        got = getattr(eng, fn)(*args, budget, **({} if shard_off is None else {"shard_off": shard_off}))
        dt = time.perf_counter() - t0
        assert got is not None, f"{fn} declined"
        _, key, pos, _, _ = np.random.get_state()
        return got[0].tolist(), got[1], (np.asarray(key).tolist(), int(pos)), dt

    for name, (ys, d, lab, c, budgets, fn) in shapes().items():
        emb, labels, av, lb = pool(ys, d, lab, 11)
        args = (emb, eng.row_norm2(emb), labels, av, lb, c)
        n = emb.shape[0]
        shard_off = [group.row_range(n, r)[0] for r in range(world)] + [n]
        call(fn, args, 50, 1, shard_off)                                  # warm-up: kernels, scratch, window
        if rank == 0:
            call(fn, args, 50, 1, None)
        for r in range(rounds):
            rec = {"shape": name, "G": world, "round": r, "n": n, "d": d, "classes": c}
            for budget in budgets:
                picks, steps, state, dt = call(fn, args, budget, 100 + r, shard_off)
                rec[f"sharded_{budget}_s"] = round(dt, 4)
                rec[f"balancing_steps_{budget}"] = steps
                everyone = [None] * world
                dist.all_gather_object(everyone, (picks, steps, state))
                rec[f"ranks_agree_{budget}"] = all(e == everyone[0] for e in everyone)
                if rank == 0:
                    p1, s1, st1, t1 = call(fn, args, budget, 100 + r, None)
                    rec[f"unsharded_{budget}_s"] = round(t1, 4)
                    rec[f"equal_to_one_gpu_{budget}"] = (p1, s1, st1) == (picks, steps, state)
                dist.barrier()
            if len(budgets) == 2:
                b1, b2 = budgets
                db = max(rec[f"balancing_steps_{b2}"] - rec[f"balancing_steps_{b1}"], 1)
                rec["sharded_ms_per_balancing_step"] = round(1e3 * (rec[f"sharded_{b2}_s"] - rec[f"sharded_{b1}_s"]) / db, 4)
                if rank == 0:
                    rec["unsharded_ms_per_balancing_step"] = round(
                        1e3 * (rec[f"unsharded_{b2}_s"] - rec[f"unsharded_{b1}_s"]) / db, 4)
            out.append(rec)
        del emb, args
        torch.cuda.empty_cache()
    if rank == 0:
        with open(out_path, "w") as f:
            json.dump(out, f)
    dist.barrier()
    eng.close()
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measures the H100 kernels and has nothing to run on a CPU")
    gpus = torch.cuda.device_count()
    print(json.dumps({"card": card(), "torch_device": torch.cuda.get_device_name(), "devices": gpus}), flush=True)
    for world in range(1, 9):
        if world > gpus:
            print(json.dumps({"G": world, "result": "not measured", "reason": f"{gpus} device(s) on this machine"}),
                  flush=True)
            continue
        with socket.socket() as sk:
            sk.bind(("127.0.0.1", 0))
            port = sk.getsockname()[1]
        path = os.path.join(tempfile.mkdtemp(prefix="alq_bal_sharded_"), "res.json")
        mp.spawn(_worker, args=(world, port, a.rounds, path), nprocs=world, join=True)
        with open(path) as f:
            for rec in json.load(f):
                print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
