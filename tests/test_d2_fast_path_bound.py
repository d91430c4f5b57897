"""The rounding bound behind the certified fast path of the D^2 draw (alq_greedy_persist.cu), checked against NumPy itself.

np.random.choice(n, p=p) returns the first k with cdf[k] > u where cdf = cumsum64(p) / its last entry and
p = fl32(c / S), c = clip(mind, 0) (float32), S = np.sum(c) (float32 pairwise).  The kernel claims: with Q the plain fp64
prefix sums of c, if Q[k] / Q_tot > u + m and Q[k-1] / Q_tot <= u - m for m = 1.3e-7, then k is NumPy's pick.  This test
draws many mass vectors (wide dynamic range, zeros, tiny and huge entries) and uniforms -- including uniforms placed
right at cdf breakpoints -- and checks that EVERY certified decision equals NumPy's, and that certification fails only
for uniforms within a few 1e-7 of a breakpoint."""
import numpy as np
import torch

from helpers import BoundaryUniforms
from oracle import al_oracle as O

MARGIN = 1.3e-7


def _certified_pick(c32, u):
    q = np.cumsum(c32.astype(np.float64))
    tot = q[-1]
    if not (tot > 0 and np.isfinite(tot)):
        return None
    r = q / tot
    k = int(np.searchsorted(r, u + MARGIN, side="right"))          # first k with Q[k]/Q_tot > u + m
    if k >= len(c32) or c32[k] <= 0:
        return None
    before = r[k - 1] if k > 0 else 0.0
    return k if before <= u - MARGIN or (k == 0 and u - MARGIN >= 0.0) or (k > 0 and before <= u - MARGIN) else None


def test_certified_decisions_equal_numpy_and_uncertain_ones_are_near_breakpoints():
    rng = np.random.default_rng(0)
    checked = uncertain = 0
    for trial in range(60):
        n = int(rng.integers(50, 6000))
        kind = trial % 4
        if kind == 0:
            c = rng.random(n).astype(np.float32) * 2000
        elif kind == 1:
            c = np.exp(rng.normal(0, 6, n)).astype(np.float32)               # 10+ orders of magnitude
        elif kind == 2:
            c = (rng.random(n) * 900).astype(np.float32)
            c[rng.random(n) < 0.4] = 0.0                                      # labeled / picked slots
        else:
            c = np.full(n, 1.0, dtype=np.float32)
            c[:: 7] = np.float32(1e-30)                                       # entries whose fl32(c/S) underflows
        lab = np.zeros(n, dtype=bool)
        p = (c / np.sum(c)).astype(np.float32)
        cdf = p.astype(np.float64).cumsum()
        cdf /= cdf[-1]
        us = list(rng.random(150))
        brk = cdf[rng.integers(0, n, 60)]
        for b in brk:                                                         # uniforms at and around breakpoints
            us += [b, np.nextafter(b, 0), np.nextafter(b, 1), b + 2e-7, b - 2e-7, b + 6e-7, b - 6e-7]
        for u in us:
            if not (0.0 <= u < 1.0):
                continue
            want = O.d2_sampling_step(c.copy(), lab, float(u))
            got = _certified_pick(c, float(u))
            if got is None:
                uncertain += 1
                assert np.min(np.abs(cdf - u)) <= 4e-7 or c[want] == 0, (trial, u)   # only near a breakpoint
            else:
                checked += 1
                assert got == want, (trial, u, got, want)
    assert checked > 8000 and uncertain > 100          # both branches were exercised


def test_callable_uniforms_equal_the_array_form():
    """`coreset_streaming` with u = f(t, cdf) picks what the array form picks when fed the values f returned, and the
    boundary schedule the GPU tests use really lands on and just beside cdf breakpoints."""
    rng = np.random.default_rng(5)
    n, l0, b = 3000, 300, 64
    for c in (0, 8):
        h = torch.from_numpy(rng.integers(-1, 2, size=(n, 16)).astype(np.float32))
        a = torch.from_numpy(rng.integers(-1, 2, size=(n, c)).astype(np.float32)) if c else None
        ind = np.zeros(n, dtype=bool)
        ind[rng.choice(n, l0, replace=False)] = True
        f = BoundaryUniforms(c, seg_end_pos=np.flatnonzero(~ind)[[99, 1999, -1]])
        cert_f, cert_a = [], []
        got = O.coreset_streaming(h, ind, b, randomize=True, uniforms=f, factors=a, certificate=cert_f)
        assert len(f.us) == b and all(0.0 <= u < 1.0 for u in f.us)
        assert got == O.coreset_streaming(h, ind, b, randomize=True, uniforms=np.array(f.us), factors=a,
                                          certificate=cert_a)
        assert cert_f == cert_a
        assert sum(x < 1e-8 for x in cert_f) >= 10
        assert sum(1.3e-7 < x <= 5e-7 for x in cert_f) >= 10


def test_uncertain_fraction_at_the_north_star_size_is_a_few_percent():
    rng = np.random.default_rng(1)
    c = (rng.random(80000) * 1500).astype(np.float32)
    us = rng.random(4000)
    frac = np.mean([_certified_pick(c, float(u)) is None for u in us])
    assert frac < 0.06, frac
