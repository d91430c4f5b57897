"""Multi-GPU selection loop vs the single-GPU loop on the same data (run under torchrun, >= 2 GPUs).
Picks must be identical for every world size: per-row arithmetic does not depend on the sharding, the arg-max key
carries the global row id, and the D^2 draw folds the same leaf sums / leaf masses in the same order on every rank.

    torchrun --nproc-per-node 2 tools/mgpu_greedy_check.py [big]

Every rank holds the full (replicated) arrays -- the engine's multi-GPU contract -- and streams only its shard."""
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from active_learning_b200.engine import Engine            # noqa: E402
from active_learning_b200.sharding import plan_shards     # noqa: E402

local = int(os.environ.get("LOCAL_RANK", "0"))
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
world, rank = dist.get_world_size(), dist.get_rank()
eng = Engine(local).comm_init()
dev = eng.device
ok = True
report = []


def case(n, l, d, c, b, ints, seed, uneven=False):
    global ok
    g = torch.Generator(device=dev).manual_seed(seed)
    if ints:
        X = torch.randint(-1, 2, (n, d), generator=g, device=dev).float()
        Y = torch.randint(-1, 2, (l, d), generator=g, device=dev).float()
        XA = torch.randint(-1, 2, (n, max(c, 4)), generator=g, device=dev).float()
        YA = torch.randint(-1, 2, (l, max(c, 4)), generator=g, device=dev).float()
    else:
        X = torch.relu(torch.randn(n, d, generator=g, device=dev))
        Y = torch.relu(torch.randn(l, d, generator=g, device=dev))
        XA = torch.randn(n, max(c, 4), generator=g, device=dev) * .05
        YA = torch.randn(l, max(c, 4), generator=g, device=dev) * .05
    fac = c > 0
    us = np.random.default_rng(seed).random(b)
    cand_pos = np.sort(np.random.default_rng(seed + 1).choice(n + l, n, replace=False)).astype(np.int32)
    vpos = torch.as_tensor(cand_pos, device=dev)
    xn, yn = eng.row_norm2(X), eng.row_norm2(Y)
    xan = eng.row_norm2(XA) if fac else None
    yan = eng.row_norm2(YA) if fac else None
    mind0 = eng.min_dist(X, xn, Y, yn, XA if fac else None, xan, YA if fac else None, yan)
    for sample in (False, True):
        single = eng.greedy_select(X, xn, mind0.clone(), [0, n], [b], a=XA if fac else None, an=xan,
                                   uniforms=us if sample else None, vpos=vpos if sample else None,
                                   full_n=[n + l] if sample else None)
        shard_off, shard_pos = plan_shards(cand_pos, n + l, world, leaf_aligned=sample)
        if uneven and not sample:
            cuts = sorted(np.random.default_rng(seed + 2).choice(np.arange(1, n), world - 1, replace=False).tolist())
            shard_off = np.asarray([0] + cuts + [n], dtype=np.int32)
        torch.cuda.synchronize()
        dist.barrier()
        t0 = time.perf_counter()
        multi, _ = eng.greedy_select(X, xn, mind0.clone(), [0, n], [b], a=XA if fac else None, an=xan,
                                     uniforms=us if sample else None, vpos=vpos if sample else None,
                                     full_n=[n + l] if sample else None, shard_off=shard_off, shard_pos=shard_pos,
                                     time_steps=True)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        tm = dict(eng.last_greedy_timing)
        same = np.array_equal(single, multi)
        allsame = torch.tensor([int(same)], device=dev)
        dist.all_reduce(allsame, op=dist.ReduceOp.MIN)
        if rank == 0:
            rec = {"n": n, "labeled": l, "d": d, "c": c, "budget": b, "integers": ints, "d2_sampling": sample,
                   "world": world, "picks_match_single_gpu": bool(allsame.item()), "wall_ms": dt * 1e3,
                   "us_per_step": dt * 1e6 / max(b - 1, 1), "stream_us": tm["stream_ms"] * 1e3, "select_us": tm["select_ms"] * 1e3}
            report.append(rec)
            print(json.dumps(rec), flush=True)
            if not allsame.item():
                k = next((i for i, (a_, b_) in enumerate(zip(single, multi)) if a_ != b_), -1)
                print("  first diff at", k, single[max(0, k - 2):k + 3], multi[max(0, k - 2):k + 3], flush=True)
        ok = ok and bool(allsame.item())


ARG = sys.argv[1] if len(sys.argv) > 1 else ""
if ARG not in ("bigonly", "tailonly", "tails"):
    case(6001, 700, 512, 0, 64, True, 1)
    case(6001, 700, 512, 40, 64, True, 2, uneven=True)
    case(3000, 300, 2048, 0, 40, False, 3)
    case(3000, 300, 2048, 1000, 40, False, 4)
if len(sys.argv) > 1 and sys.argv[1] in ("big", "bigonly"):
    case(80000, 50000, 2048, 0, 2000, False, 5)
    case(80000, 50000, 2048, 1000, 2000, False, 6)


def tail_case(n_per, c, b, seed, dyadic=False):
    """K1 + K1b + exchange as one launch per rank vs one GPU on the concatenated pool (uneven shards too)."""
    global ok
    g = torch.Generator(device=dev).manual_seed(seed)
    sizes = [n_per + (37 * q if seed % 2 else 0) for q in range(world)]
    n_tot = sum(sizes)
    if dyadic:
        logits = torch.randint(-2, 3, (n_tot, c), generator=g, device=dev).float()
    else:
        logits = torch.randn(n_tot, c, generator=g, device=dev) * 3
    lo = sum(sizes[:rank])
    shard = logits[lo:lo + sizes[rank]].contiguous()
    for mode in (0, 1, 2):
        _, ref = eng.uncertainty_tail(logits, mode, b)
        torch.cuda.synchronize()
        dist.barrier()
        _, got = eng.uncertainty_tail_sharded(shard, mode, b, lo, min(sizes), max(sizes))
        torch.cuda.synchronize()
        try:
            eng.comm_check()
        except Exception as exc:              # e.g. a tie group beyond the window regions: reported, never silent
            if rank == 0:
                print(json.dumps({"tail": True, "rows_per_rank": sizes, "c": c, "budget": b, "mode": mode, "fused_path_reported": str(exc)[:120]}), flush=True)
            continue
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        dist.barrier()
        e0.record()
        for _ in range(20):
            eng.uncertainty_tail_sharded(shard, mode, b, lo, min(sizes), max(sizes))
        e1.record()
        torch.cuda.synchronize()
        same = torch.tensor([int(torch.equal(ref, got))], device=dev)
        dist.all_reduce(same, op=dist.ReduceOp.MIN)
        if rank == 0:
            rec = {"tail": True, "rows_per_rank": sizes, "c": c, "budget": b, "mode": mode, "dyadic": dyadic, "world": world,
                   "picks_match_single_gpu": bool(same.item()), "us_per_call": e0.elapsed_time(e1) * 1e3 / 20}
            report.append(rec)
            print(json.dumps(rec), flush=True)
        ok = ok and bool(same.item())


if ARG != "tailonly":
    tail_case(20000, 1000, 10000, 11)
    tail_case(9000, 64, 3000, 12, dyadic=True)
    tail_case(4200, 1000, 700, 13)
if ARG in ("big", "bigonly", "tailonly", "tails"):
    tail_case(80000, 1000, 10000, 14)
dist.barrier()
if rank == 0:
    print("MGPU GREEDY", "PASS" if ok else "FAIL", flush=True)
    out = os.environ.get("ALQ_CHECK_OUT", tempfile.gettempdir())
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, f"mgpu_greedy_check_n{world}.json"), "w") as fh:
        json.dump({"pass": ok, "cases": report}, fh, indent=1)
dist.destroy_process_group()
sys.exit(0 if ok else 1)
