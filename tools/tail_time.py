"""Headline tail (K1 + K1b) timing on one GPU: fused cooperative launch vs the two separate kernels. JSON lines."""
import json, os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from active_learning_b200.engine import Engine
eng = Engine(0)
g = torch.Generator(device="cuda").manual_seed(0)
N, C, B = 80000, 1000, 10000
HBM_BYTES_PER_S = 3.35e12       # H100 SXM data sheet (a card below 700 W may not reach it)
logits = torch.randn(N, C, device="cuda", generator=g) * 3
scores = torch.empty(N, device="cuda")
def timeit(fn, reps=50):
    for _ in range(5): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / reps
for mode in (0, 1, 2):
    fused = timeit(lambda: eng.uncertainty_tail(logits, mode, B, scores_out=scores))
    stream_ms, kernel_ms = eng.uncertainty_tail_timing()     # the last fused launch, from its %globaltimer stamps
    def two():
        eng.score_softmax(logits, mode, out=scores); eng.select_smallest(scores, B)
    sep = timeit(two)
    k1 = timeit(lambda: eng.score_softmax(logits, mode, out=scores))
    print(json.dumps({"mode": mode, "fused_us": round(fused, 2), "separate_us": round(sep, 2), "k1_alone_us": round(k1, 2),
                      "fused_frac_of_datasheet_hbm": round(N * (4 * C + 4) / (fused * 1e-6) / HBM_BYTES_PER_S, 4),
                      "fused_stream_ms": round(stream_ms, 4), "fused_kernel_ms": round(kernel_ms, 4),
                      "gpu": torch.cuda.get_device_name(0)}), flush=True)
