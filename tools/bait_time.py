"""BAITSampler on the H100: K24 (the Fisher), K25 (the initial forms) and K26's three passes (labeled absorption, forward,
backward) timed with CUDA events, and a few steps of the authors' literal per-step formulation in torch fp64 on the same
card for comparison (every candidate's C x (C D) matrix V_x materialised, Vt A, Vt A F A Vt^T and (I + Vt A Vt^T)^-1 at
every step), measured, not extrapolated.

    python tools/bait_time.py [--shapes NxD:L:B,...] [--classes C] [--literal-steps K]

A shape NxD:L:B is n pool rows of width D, L labeled rows and budget B (default CIFAR-10's 50 000 rows at D = 512 and
2 048, 5 000 labeled, B = 1 000).  Prints the card, its power limit and max SM clock first, then one JSON line per shape.
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


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:            # noqa: BLE001
        return f"unknown ({e})"


def events(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return out, a.elapsed_time(b)


def pool(n, d, c, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    h = torch.randn(n, d, device="cuda", generator=g)
    w = torch.randn(d, c, device="cuda", generator=g) * (3.0 / d ** 0.5)
    return (h @ w + 0.5 * torch.randn(n, c, device="cuda", generator=g)).contiguous(), h


def literal_steps(p, h, F, A, cand, s, steps, chunk=2048):
    """The authors' step: for every candidate tr(Vt A F A Vt^T (I + Vt A Vt^T)^-1) with Vt materialised, the argmax, then
    A's update.  Returns the per-step milliseconds (CUDA events, each step synchronised)."""
    c = p.shape[1]
    eye = torch.eye(c, dtype=torch.float64, device="cuda")
    out = []
    for _ in range(steps):
        t0 = torch.cuda.Event(enable_timing=True)
        t1 = torch.cuda.Event(enable_timing=True)
        t0.record()
        best, arg = -float("inf"), -1
        AF = A @ F
        for lo in range(0, len(cand), chunk):
            rows = cand[lo:lo + chunk]
            px = p[rows]
            R = torch.sqrt(px)[:, :, None] * (eye[None] - px[:, None, :])
            V = s * (R[:, :, :, None] * h[rows].double()[:, None, None, :]).reshape(len(rows), c, -1)
            VA = V @ A
            inner = torch.linalg.inv(eye[None] + VA @ V.transpose(1, 2))
            score = torch.diagonal((VA @ AF.T) @ V.transpose(1, 2) @ inner, dim1=1, dim2=2).sum(-1)
            v, i = score.max(dim=0)
            if float(v) > best:
                best, arg = float(v), int(rows[int(i)])
        px = p[arg]
        R = torch.sqrt(px)[:, None] * (eye - px[None, :])
        Vx = s * torch.kron(R, h[arg].double()[None, :])
        VA = Vx @ A
        A = A - VA.T @ torch.linalg.inv(eye + VA @ Vx.T) @ VA
        t1.record()
        torch.cuda.synchronize()
        out.append(t0.elapsed_time(t1))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="50000x512:5000:1000,50000x2048:5000:1000")
    ap.add_argument("--classes", type=int, default=10)
    ap.add_argument("--literal-steps", type=int, default=2)
    args = ap.parse_args()
    from active_learning_b200.engine import Engine
    print("card:", card(), flush=True)
    eng = Engine()
    c = args.classes
    for spec in args.shapes.split(","):
        nd, n_lab, budget = spec.split(":")
        n, d = (int(v) for v in nd.split("x"))
        n_lab, budget = int(n_lab), int(budget)
        eng.bait_guard(n, c, d)
        z, h = pool(n, d, c, n + d)
        rng = np.random.default_rng(0)
        is_lab = np.zeros(n, dtype=bool)
        is_lab[rng.choice(n, n_lab, replace=False)] = True
        lab, cand = np.flatnonzero(is_lab), np.flatnonzero(~is_lab)
        eng.bait_fisher(z[:256], h[:256])                              # loads the module
        (p, F), t_fisher = events(lambda: eng.bait_fisher(z, h))
        state, t_init = events(lambda: eng.bait_init(h, F, 1.0))
        phase = np.zeros(3, dtype=np.float32)
        t0 = time.perf_counter()
        picks, order, fwd, bwd = eng.bait_select(h, p, F, state, lab, cand, budget, phase_ms=phase)
        wall = time.perf_counter() - t0
        del state
        T = len(order)
        rec = {"n": n, "d": d, "c": c, "labeled": n_lab, "budget": budget, "dim": c * d,
               "fisher_ms": round(t_fisher, 2), "init_ms": round(t_init, 2),
               "absorb_ms": round(float(phase[0]), 1), "forward_ms": round(float(phase[1]), 1),
               "backward_ms": round(float(phase[2]), 1),
               "absorb_step_ms": round(float(phase[0]) / max(n_lab, 1), 3),
               "forward_step_ms": round(float(phase[1]) / max(T, 1), 3),
               "backward_step_ms": round(float(phase[2]) / max(T - budget, 1), 3),
               "select_wall_s": round(wall, 2), "picks": len(picks), "distinct": len(set(picks.tolist()))}
        if args.literal_steps > 0:
            # the literal loop from the same A the forward pass starts from: M0 densely inverted
            from_lab = torch.from_numpy(lab).cuda()
            s_lab = 1.0 / np.sqrt(n_lab + budget)
            s = float(np.sqrt(budget / (n_lab + budget)))
            M = torch.eye(c * d, dtype=torch.float64, device="cuda")
            hd = h[from_lab].double()
            for a in range(c):
                for b in range(a, c):
                    w = ((p[from_lab, a] if a == b else 0.0) - p[from_lab, a] * p[from_lab, b]) * s_lab ** 2
                    blk = hd.T @ (w[:, None] * hd)
                    M[a * d:(a + 1) * d, b * d:(b + 1) * d] += blk
                    if a != b:
                        M[b * d:(b + 1) * d, a * d:(a + 1) * d] += blk.T
            A = torch.linalg.inv(M)
            del M, hd
            lit = literal_steps(p, h, F, A, torch.from_numpy(cand).cuda(), s, args.literal_steps)
            rec["literal_step_ms"] = [round(v, 1) for v in lit]
            del A
        print(json.dumps(rec), flush=True)
        del p, F
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
