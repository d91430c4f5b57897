"""VAALSampler's query on the H100: K9 (the discriminator on the tensor cores) + K1b timed with CUDA events, and the
whole query against the reference's loop (tests/vaal_oracle.py: the full VAE per batch, `.cpu()` per batch, topk on the
host) on the same GPU, modules and pool, the two arms alternated in one run.

    python tools/vaal_time.py [--sizes 80000 1240000] [--z 64] [--pool 20000] [--out FILE]

K9's rate counts the 3xTF32 issue, 3 * 2 * N * (z * 512 + 512 * 512 + 512) flop, against cuBLAS's TF32 GEMM measured in
the same run (8192^3, best of 10), as DESIGN.md section 4 does for K3.  The end-to-end pool is `--pool` images of
3 x 224 x 224 (a bank of 1000 seeded images, each item offset by its index so that no two are equal), C = 1000
(latent_scale 2), batch 128, budget 10 % of the pool; the modules carry the seeded weights of tests/vaal_oracle.py.
cuDNN and cuBLAS run with torch's defaults in both arms.  Prints one JSON line per measurement, the card's name and
power limit first.
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
import vaal_oracle as V  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:            # noqa: BLE001
        q = f"unknown ({e})"
    return q


def events_ms(fn, repeats):
    out = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return out


def cublas_tf32_tflops():
    saved = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    a = torch.randn(8192, 8192, device="cuda")
    b = torch.randn(8192, 8192, device="cuda")
    for _ in range(3):
        a @ b
    best = min(events_ms(lambda: a @ b, 10))
    torch.backends.cuda.matmul.allow_tf32 = saved
    return 2 * 8192 ** 3 / best / 1e9


class ImageBank(torch.utils.data.Dataset):
    def __init__(self, n, num_classes, seed=0):
        self.n, self.num_classes, self.targets = n, num_classes, [0] * n
        self.bank = torch.from_numpy(np.random.default_rng(seed).standard_normal((1000, 3, 224, 224)).astype(np.float32))

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        return self.bank[i % 1000] + i * 1e-3, 0, i


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="*", default=[80000, 1240000])
    ap.add_argument("--z", type=int, default=64)
    ap.add_argument("--budget", type=int, default=10000)
    ap.add_argument("--pool", type=int, default=20000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from active_learning_b200.engine import Engine
    from active_learning_b200.query_strategies.get_strategy import get_strategy
    eng = Engine()
    results = [{"card": card(), "torch_device": torch.cuda.get_device_name()}]
    print(json.dumps(results[0]), flush=True)
    peak = cublas_tf32_tflops()
    results.append({"cublas_tf32_gemm_8192_tflops": round(peak, 1)})
    print(json.dumps(results[-1]), flush=True)

    disc = V.seeded_state(V.Discriminator(z_dim=args.z), 7).cuda()
    for n in args.sizes:
        g = torch.Generator(device="cuda").manual_seed(n)
        mu = torch.randn(n, args.z, device="cuda", generator=g)
        b = min(args.budget, n)
        eng.select_smallest(eng.vaal_scores(mu, disc), b)            # warm-up: module load, scratch
        torch.cuda.synchronize()
        k9 = events_ms(lambda: eng.vaal_scores(mu, disc), 10)
        tail = events_ms(lambda: eng.select_smallest(eng.vaal_scores(mu, disc), b), 10)
        flop = 3 * 2.0 * n * (args.z * 512 + 512 * 512 + 512)
        k9_med = float(np.median(k9))
        rec = {"n": n, "z": args.z, "budget": b, "k9_ms_min_med_max": [round(min(k9), 3), round(k9_med, 3), round(max(k9), 3)],
               "k9_plus_k1b_ms_min_med_max": [round(min(tail), 3), round(float(np.median(tail)), 3), round(max(tail), 3)],
               "k9_tf32_tflops": round(flop / k9_med / 1e9, 1), "k9_share_of_cublas_tf32": round(flop / k9_med / 1e9 / peak, 3)}
        results.append(rec)
        print(json.dumps(rec), flush=True)
        del mu

    # ---- end to end: the reference's loop against the sampler, same GPU, modules and pool, alternated
    ds = ImageBank(args.pool, 1000)
    vae = V.seeded_state(V.VAE(z_dim=args.z, nc=3, latent_scale=2), 8).cuda()
    vae.set_crop_seed(1234)
    budget = args.pool // 10
    net = torch.nn.Linear(4, 1000)
    kw = dict(early_stop_patience=0, n_epoch=1, world_size=1, model="SSLResNet18", freeze_feature=False,
              ckpt_path=tempfile.mkdtemp(prefix="vaal_time_"), exp_name="t", vae=vae, discriminator=disc)
    s = get_strategy("VAALSampler")(ds, ds, net, {"loader_te_args": {"batch_size": 128, "num_workers": 0}},
                                    np.array([], dtype=np.int64), None, None, **kw)
    s.set_engine(eng)

    def ours():
        np.random.seed(5)
        return s.query(float(budget))[0]

    def reference():
        np.random.seed(5)
        cand = s.available_query_idxs()
        return V.reference_query(ds, cand, 128, vae, disc, float(budget), device="cuda")[0]

    times = {"reference": [], "engine": []}
    picks = {}
    for rep in range(args.repeats + 1):                               # the first round is the warm-up
        for name, fn in (("reference", reference), ("engine", ours)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            picks[name] = np.asarray(fn())
            torch.cuda.synchronize()
            if rep:
                times[name].append(time.perf_counter() - t0)
    a, b_ = picks["reference"], picks["engine"]
    rec = {"pool": args.pool, "image": [3, 224, 224], "batch": 128, "budget": budget, "repeats": args.repeats,
           "reference_s": [round(t, 3) for t in times["reference"]], "engine_s": [round(t, 3) for t in times["engine"]],
           "speedup_median": round(float(np.median(times["reference"]) / np.median(times["engine"])), 2),
           "pick_set_agreement": round(len(np.intersect1d(a, b_)) / budget, 4),
           "pick_order_identical": bool(np.array_equal(a, b_))}
    results.append(rec)
    print(json.dumps(rec), flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(results, fh, indent=1)


if __name__ == "__main__":
    main()
