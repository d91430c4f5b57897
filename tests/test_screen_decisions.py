"""K15's and K18's screen decisions without a GPU: why K15 refuses norms outside its band's domain, K15's band inside
that domain under the three emulated adders, K18's fp32 round-down of its lower bounds, and K18's fallback decision
(cal_oracle.fallback_decide) against brute force.  test_gpu_screen_decisions.py predicts both kernels' decisions from
the H100's own dot products with these helpers."""
import itertools
from fractions import Fraction

import numpy as np
import pytest

import cal_oracle as CO
import probcover_oracle as P
import typiclust_oracle as T


def k15_counterexample():
    """A zero row against centre 0 = a (a = 1e3 N(0, 1) in fp32, d = 64) and centre 1 = a permutation of a: g = 0 and
    nrm2 = 0 exactly on any card, so K15's decision depends only on the lane-ordered cn.  At |c|^2 ~ 6e7 an fp64 ulp
    exceeds the slack 1e-9, so cn +- 1e-9 rounds back to cn, and the band certifies the smaller lane-ordered cn while the
    exact (sequential) sums order the two centres the other way.  Returns (zero row [1, 64], centres [2, 64])."""
    rng = np.random.default_rng(0)
    a = (1e3 * rng.normal(size=64)).astype(np.float32)
    cen = np.stack([a, a[rng.permutation(64)]])
    return np.zeros((1, 64), dtype=np.float32), cen


def test_k15_certifies_the_wrong_centre_outside_its_domain():
    x, cen = k15_counterexample()
    cn = P.nrm2(cen)
    assert (cn > 2.0).all()
    decided, c1 = T.assign_decide(64, P.nrm2(x), cn, np.zeros((1, 2), dtype=np.float32))
    assert decided[0] and c1[0] == 1
    assert T.exact_argmin(x, cen)[0] == 0
    e = P.exact_d2(np.repeat(x, 2, axis=0), cen)
    assert e[0] < e[1]                                                   # a strict order, not a tie to the lower centre
    assert (cn + 1e-9 == cn).all() and (cn - 1e-9 == cn).all()          # the slack vanishes in the rounding


def test_exact_argmin_is_brute_force_with_ties_to_the_lowest_centre():
    rng = np.random.default_rng(3)
    x = rng.normal(size=(300, 12)).astype(np.float32) * 50
    c = rng.normal(size=(40, 12)).astype(np.float32) * 50
    c[7] = c[30]                                                         # an exact tie: the lower centre
    x[:10] = c[30]
    got = T.exact_argmin(x, c, chunk=64)
    i, j = np.meshgrid(np.arange(300), np.arange(40), indexing="ij")
    d2 = P.exact_d2(x[i.ravel()], c[j.ravel()]).reshape(300, 40)
    assert got.tolist() == np.argmin(d2, axis=1).tolist()
    assert (got[:10] == 7).all()


def _pushed(rows, to=2.0):
    """fp32 rows scaled so that their lane-ordered nrm2 lies just below `to` (zero rows stay zero)."""
    rows = np.asarray(rows, dtype=np.float32)
    n2 = P.nrm2(rows)
    s = np.where(n2 > 0, np.sqrt(to / np.where(n2 > 0, n2, 1.0)) * (1 - 2.0 ** -20), 1.0)
    out = (rows.astype(np.float64) * s[:, None]).astype(np.float32)
    assert (P.nrm2(out) <= to).all()
    return out


@pytest.mark.parametrize("d", [4, 28, 64, 520, 2048])
def test_k15_band_holds_at_the_edge_of_its_domain(d):
    """Rows and centres pushed to nrm2 = 2 (the domain's edge; antipodes give d2 = 8), under the three adder models:
    |d2~ - exact_d2| <= K15's b for every pair, and every row the band decides gets the brute-force argmin."""
    rng = np.random.default_rng(300 + d)
    fam = P.bound_families(rng, d, instances=2)
    xh = _pushed(np.concatenate(list(fam.values())))
    picks = [rng.choice(len(xh), int(rng.integers(2, 9)), replace=False) for _ in range(16)]
    cen = np.stack([xh[p].astype(np.float64).mean(axis=0) for p in picks]).astype(np.float32)
    cen = np.concatenate([_pushed(cen), -xh[:6], xh[7:8], np.zeros((1, d), dtype=np.float32)])
    nx, cn = P.nrm2(xh), P.nrm2(cen)
    assert nx.max() > 1.99 and cn.max() > 1.99 and max(nx.max(), cn.max()) <= 2.0
    i, j = np.meshgrid(np.arange(len(xh)), np.arange(len(cen)), indexing="ij")
    i, j = i.ravel(), j.ravel()
    e = P.exact_d2(xh[i], cen[j])
    assert e.max() > 7.9
    coef = 2.0 * P.screen_bound(d, 1.0, 1.0) * (1.0 + 1e-6)
    b = coef * (np.sqrt(nx[i]) * np.sqrt(cn[j])) + 1e-9
    want = T.exact_argmin(xh, cen)
    for adder in ("nearest", "zero", "align"):
        g = P.emulate_3xtf32(xh[i], cen[j], adder=adder)
        d2 = (nx[i] + cn[j]) - 2.0 * g.astype(np.float64)
        assert (np.abs(d2 - e) <= b).all(), adder
        ok, c1 = T.assign_decide(d, nx, cn, g.reshape(len(xh), len(cen)))
        assert (c1[ok] == want[ok]).all() and ok.any(), adder


# ---- K18's fp32 lower bounds -------------------------------------------------------------------------------------------
def _rd_by_definition(v):
    """The largest fp32 value f <= v (exact rationals), as __double2float_rd is defined; -inf below -FLT_MAX."""
    out = []
    with np.errstate(over="ignore"):
        for x in np.asarray(v, dtype=np.float64):
            f = np.float32(x)                                            # to nearest: within one fp32 step of the answer
            for cand in (np.nextafter(f, np.float32(np.inf)), f, np.nextafter(f, np.float32(-np.inf))):
                if np.isfinite(cand) and Fraction(float(cand)) <= Fraction(float(x)):
                    nxt = np.nextafter(cand, np.float32(np.inf))
                    if not np.isfinite(nxt) or Fraction(float(nxt)) > Fraction(float(x)):
                        out.append(cand)
                        break
            else:
                out.append(np.float32(-np.inf))
    return np.asarray(out, dtype=np.float32)


def test_f32_round_down():
    rng = np.random.default_rng(9)
    f32 = np.concatenate([rng.normal(size=200), [0.0, -0.0, 1.0, -1.0, 2.0 ** -149, -(2.0 ** -149), 2.0 ** -126,
                                                 float(np.finfo(np.float32).max)]]).astype(np.float32)
    assert (CO._f32_down(f32.astype(np.float64)).view(np.uint32) == f32.view(np.uint32)).all()   # exact: unchanged
    f = np.abs(rng.normal(size=300)).astype(np.float32) + np.float32(1e-3)
    nxt = np.nextafter(f, np.float32(np.inf))
    for w in (0.25, 0.5, 0.75, 1e-9):                                    # between two fp32 values: the lower
        mid = f.astype(np.float64) + w * (nxt.astype(np.float64) - f.astype(np.float64))
        assert (CO._f32_down(mid) == f).all()
        assert (CO._f32_down(-mid) == -nxt).all()                        # negative: away from zero
    tiny = np.array([1e-50, -1e-50, 2.0 ** -150, -(2.0 ** -150), 3 * 2.0 ** -151, 2.0 ** -140 * 1.3, -(2.0 ** -140) * 1.3])
    want = np.array([0.0, -1, 0.0, -1, 0, 665, -666]) * 2.0 ** -149   # steps of 2^-149: 0.75 -> 0, 1.3 * 2^9 -> 665
    assert (CO._f32_down(tiny).astype(np.float64) == want).all()
    big = np.array([3.5e38, -3.5e38, 1e300])
    assert CO._f32_down(big).tolist() == [float(np.finfo(np.float32).max), -np.inf, float(np.finfo(np.float32).max)]
    v = np.concatenate([rng.normal(size=300) * 10.0 ** rng.uniform(-45, 38, 300), tiny, big, -big])
    assert (CO._f32_down(v).view(np.uint32) == _rd_by_definition(v).view(np.uint32)).all()


def test_screen_lower_is_a_lower_bound_in_the_kernels_order():
    rng = np.random.default_rng(10)
    for d in (28, 2048):
        nx = 10.0 ** rng.uniform(-6, 6, 50)
        ny = 10.0 ** rng.uniform(-6, 6, 40)
        g = (rng.uniform(-1, 1, (50, 40)) * np.sqrt(nx[:, None] * ny[None, :])).astype(np.float32)
        L = CO.screen_lower(d, nx[:, None], ny[None, :], g)
        v = CO.screen_d2(nx[:, None], ny[None, :], g) - CO.band(d, nx[:, None], ny[None, :])
        assert L.dtype == np.float32
        assert (L.astype(np.float64) <= v).all()
        assert (np.nextafter(L, np.float32(np.inf)).astype(np.float64) > v).all()


# ---- K18's fallback decision -------------------------------------------------------------------------------------------
def _exact_from(E):
    return lambda r, c: E[r, c]


def _brute(Lrow, Erow, k):
    """Every decision a kept set of the S smallest bounds (any choice among those tied at the boundary) gives."""
    m = len(Lrow)
    if m <= CO.S_KEPT:
        return {False}
    srt = np.sort(Lrow)
    edge, lstar = srt[CO.S_KEPT - 1], srt[CO.S_KEPT]
    sure = np.flatnonzero(Lrow < edge)
    tied = np.flatnonzero(Lrow == edge)
    out = set()
    for pick in itertools.combinations(tied, CO.S_KEPT - len(sure)):
        kept = np.concatenate([sure, np.asarray(pick, dtype=np.int64)])
        o = np.lexsort((kept, Erow[kept]))
        out.add(bool(float(lstar) <= Erow[kept][o][k - 1]))
    return out


def _lists(Lrow, Erow, k, order):
    """K18's lists_offer literally, the columns offered in `order`: (L*, the decision)."""
    kept, ls = [], np.float32(np.inf)
    for c in order:
        v = Lrow[c]
        thr = max(Lrow[q] for q in kept) if len(kept) == CO.S_KEPT else np.float32(np.inf)
        if not v < thr:
            ls = min(ls, v)
            continue
        if len(kept) == CO.S_KEPT:
            a = max(range(CO.S_KEPT), key=lambda q: (Lrow[kept[q]], -q))  # the first position of the largest
            ls = min(ls, Lrow[kept[a]])
            kept[a] = c
        else:
            kept.append(c)
    kept = np.asarray(kept)
    ek = np.sort(Erow[kept])[k - 1] if len(kept) >= k else np.inf
    return ls, not (ls == np.inf or ls > ek)


@pytest.mark.parametrize("k", [1, 10, 32])
def test_fallback_decide_against_brute_force(k):
    rng = np.random.default_rng(20 + k)
    # While every L is a lower bound of its exact value, a tie at the boundary never changes the decision: the columns
    # below L* = t are the same whichever tied one is kept, and each tied one has exact >= t.  A broken bound can:
    # 31 bounds certainly kept (exact 50), two tied at L* = 40 with exact 30 (below its bound) and 100.  Keeping the
    # first gives E_1 = 30 < 40 (no fallback), the second E_1 = 50 (a fallback); E_10, E_32 = 50 fall back either way.
    L0 = np.concatenate([np.arange(31), [40, 40]]).astype(np.float32)[None]
    E0 = np.concatenate([np.full(31, 50.0), [30.0, 100.0]])[None]
    two = {False, True} if k == 1 else {True}
    assert CO.fallback_decide(L0, _exact_from(E0), k)[0] == two == _brute(L0[0], E0[0], k)
    for m in (5, 31, 32, 33, 34, 40, 70):
        for trial in range(12):
            E = np.round(rng.uniform(0, 4, size=(1, m)), 1)              # exact d2 with ties
            L = (E - rng.choice([0.0, 0.05, 0.2, 0.5], size=(1, m))).astype(np.float32)
            if trial % 3 == 0:                                           # ties at the 32 / 33 boundary
                srt = np.sort(L[0])
                if m > CO.S_KEPT:
                    L[0, np.abs(L[0] - srt[CO.S_KEPT]) < 0.3] = srt[CO.S_KEPT]
            if trial % 3 == 1 and m > CO.S_KEPT:                         # L* right at E_k: L* <= E_k falls back
                o = np.argsort(L[0], kind="stable")
                E[0, o[:CO.S_KEPT]] = np.maximum(E[0, o[:CO.S_KEPT]], L[0, o[:CO.S_KEPT]])
                ek = np.sort(E[0, o[:CO.S_KEPT]])[k - 1]
                L[0, o[CO.S_KEPT:]] = np.maximum(L[0, o[CO.S_KEPT:]], np.float32(ek))
                L[0, o[CO.S_KEPT]] = np.float32(ek) if np.float32(ek) == ek else L[0, o[CO.S_KEPT]]
            got = CO.fallback_decide(L, _exact_from(E), k)[0]
            assert set(got) == _brute(L[0], E[0], k), (m, trial)
            srt = np.sort(L[0])
            for _ in range(3):
                ls, dec = _lists(L[0], E[0], k, rng.permutation(m))
                assert ls == (srt[CO.S_KEPT] if m > CO.S_KEPT else np.inf)
                assert dec in got
            if m <= CO.S_KEPT:
                assert got == {False}
            assert len(got) == 1 or (L > E).any()                        # while the bounds hold: one decision


def test_fallback_decide_asks_only_for_the_kept_columns():
    rng = np.random.default_rng(5)
    L = np.stack([rng.permutation(300) * np.float32(0.125) for _ in range(6)]).astype(np.float32)
    E = L.astype(np.float64) + 0.01                                      # L* = E_32 - 0.01 + 0.125: no fallback
    asked = []

    def exact(r, c):
        asked.append(len(r))
        return E[r, c]
    dec = CO.fallback_decide(L, exact, 32)
    assert asked == [6 * 32] and all(d == {False} for d in dec)
    L[:, 5] = np.sort(L, axis=1)[:, 32] - 1                              # a 33rd bound below E_32: every row falls back
    dec = CO.fallback_decide(L, _exact_from(E), 32)
    assert all(d == {True} for d in dec)
