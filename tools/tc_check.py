"""K3 tensor-core path vs the exact SIMT path / torch, with timings (bring-up aid of the wgmma kernel)."""
import sys, os, time
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from active_learning_b200.engine import Engine

eng = Engine(0)
torch.manual_seed(0)

def run(n, m, d, c=0, ints=False, red_max=False):
    g = torch.Generator(device="cuda").manual_seed(n + m + d)
    if ints:
        x = torch.randint(-1, 2, (n, d), device="cuda", generator=g).float()
        y = torch.randint(-1, 2, (m, d), device="cuda", generator=g).float()
    else:
        x = torch.relu(torch.randn(n, d, device="cuda", generator=g))
        y = torch.relu(torch.randn(m, d, device="cuda", generator=g))
    xa = ya = xan = yan = None
    if c:
        if ints:
            xa = torch.randint(-1, 2, (n, c), device="cuda", generator=g).float()
            ya = torch.randint(-1, 2, (m, c), device="cuda", generator=g).float()
        else:
            xa = torch.randn(n, c, device="cuda", generator=g) * 0.05
            ya = torch.randn(m, c, device="cuda", generator=g) * 0.05
        xan, yan = eng.row_norm2(xa), eng.row_norm2(ya)
    xn, yn = eng.row_norm2(x), eng.row_norm2(y)
    res = {}
    for impl in (1, 2):
        eng.set_option("k3_impl", impl)
        torch.cuda.synchronize()
        out = eng.min_dist(x, xn, y, yn, xa, xan, ya, yan, reduce_max=red_max)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = eng.min_dist(x, xn, y, yn, xa, xan, ya, yan, reduce_max=red_max)
        torch.cuda.synchronize()
        res[impl] = (out, (time.perf_counter() - t0) * 1e3)
    eng.set_option("k3_impl", 0)
    a, b = res[1][0], res[2][0]
    scale = float((xn.max() * (xan.max() if c else 1)) + (yn.max() * (yan.max() if c else 1)))
    err = float((a - b).abs().max())
    flop = 2.0 * n * m * (d + c)
    print(f"n={n} m={m} d={d} c={c} ints={ints} max={red_max}: simt {res[1][1]:.2f} ms ({flop/res[1][1]/1e9:.1f} TF)  "
          f"tc {res[2][1]:.2f} ms ({flop/res[2][1]/1e9:.1f} TF)  max|diff|={err:.3e} rel={err/scale:.2e} "
          f"{'EXACT' if torch.equal(a, b) else ''}", flush=True)
    return err / scale

which = sys.argv[1] if len(sys.argv) > 1 else "small"
if which == "small":
    run(128, 256, 32, ints=True)
    run(128, 256, 64, ints=True)
    run(300, 700, 96, ints=True)
    run(1000, 1000, 2048, ints=True)
    run(1000, 1000, 2048)
    run(777, 1313, 516, red_max=True)
    run(500, 600, 64, c=40, ints=True)
    run(500, 600, 2048, c=1000)
else:
    run(20000, 10000, 2048, ints=True)
    run(80000, 50000, 2048)
    run(80000, 50000, 2048, c=1000)
print("tc_check done")
