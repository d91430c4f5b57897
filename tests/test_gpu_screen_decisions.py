"""K15's and K18's certified screens held to the H100's own tensor cores: every decision predicted from the hardware's dot
products, at band edges to one ulp, and K18's band across its whole norm range; K15 refuses norms outside its band's
domain.

g is read through K3 (`gram_hw` of test_gpu_tf32_bound.py, exact by construction).  K15 and K18 issue the same chain
(tc::ring_tile), and test_gpu_tf32_bound.py shows that a pair's g does not depend on its place in the tile, so the
epilogues' fp64 arithmetic (typiclust_oracle.assign_decide, cal_oracle.screen_lower / fallback_decide) applied to K3's g
predicts each kernel's recheck and fallback counts row by row.  A row at a band edge flips on one ulp of one coordinate,
so a band half or twice as wide, or a wrong order in the epilogue, changes a count.
"""
import numpy as np
import pytest
import torch

import cal_oracle as CO
import probcover_oracle as P
import typiclust_oracle as T
from test_gpu_cal import _rows
from test_gpu_tf32_bound import gram_hw
from test_gpu_typiclust import _centres, _clustered
from test_screen_decisions import k15_counterexample

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from active_learning_b200.engine import Engine
    return Engine()


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def _unit(rng, n, d):
    return T.normalize(rng.normal(size=(n, d)).astype(np.float32))


def _with_bits(v, j, bits):
    """v with coordinate j set to the fp32 of bit pattern `bits`."""
    out = np.array(v, dtype=np.float32, copy=True)
    out[j] = np.array([bits], dtype=np.int32).view(np.float32)[0]
    return out


def _edge(dec, lo, hi):
    """Adjacent integer bit patterns p, p + 1 between lo and hi with dec(p) != dec(p + 1), by bisection from
    dec(lo) != dec(hi) (no monotonicity needed)."""
    dlo, dhi = dec(lo), dec(hi)
    assert dlo != dhi
    while hi - lo > 1:
        mid = (lo + hi) // 2
        dm = dec(mid)
        if dm == dlo:
            lo = mid
        else:
            hi, dhi = mid, dm
    return lo, hi


# ---- A. K15's recheck count predicted row by row -----------------------------------------------------------------------
@pytest.mark.parametrize("K", [1, 2, 129, 500])
@pytest.mark.parametrize("d", [28, 64, 520, 2048])
def test_k15_rechecks_the_rows_its_band_predicts(eng, d, K):
    """Clustered unit rows against means of them with exact ties and one-ulp copies: K15's recheck count equals the
    count assign_decide gives from K3's g, every row the band decides gets c1, and every label is the brute-force
    argmin.  At K = 1 the second bound is +inf and nothing is rechecked."""
    rng = np.random.default_rng(31 * d + K)
    n = 1037                                                            # a partial last row tile
    xhat = T.normalize(_clustered(n, d, 24, d + K))
    cen = _centres(rng, xhat, K)
    G = gram_hw(eng, xhat, cen)
    decided, c1 = T.assign_decide(d, P.nrm2(xhat), P.nrm2(cen), G)
    want = T.exact_argmin(xhat, cen)
    labels, changed, rech = eng.kmeans_assign(_cuda(xhat), _cuda(cen))
    assert rech == int((~decided).sum()), (d, K, rech, int((~decided).sum()))
    assert (c1[decided] == want[decided]).all()
    assert labels.cpu().numpy().tolist() == want.tolist() and changed == n
    if K == 1:
        assert rech == 0
    if K >= 8:
        assert 0 < rech < n


# ---- B. K15 at its band edge, to one ulp -------------------------------------------------------------------------------
def _k15_case(rng, d, K):
    """A unit row x, a centre c_a near it, K far unit centres, and the row's g against them."""
    x = _unit(rng, 1, d)[0]
    ca = T.normalize((x + 0.15 * rng.normal(size=d) / np.sqrt(d)).astype(np.float32)[None])[0]
    far = _unit(rng, K, d)
    return x, ca, far


@pytest.mark.parametrize("d", [64, 520])
def test_k15_decides_at_its_band_edge(eng, d):
    """c_b = c_a with one coordinate bisected over its fp32 bit patterns until adjacent patterns decide differently
    (assign_decide on K3's g); at both patterns K15's recheck count and labels equal the prediction, for the row alone
    and at positions 0, 127, 128 and 1036 of a 1037-row pool, with c_b in c_a's centre tile, in a later tile, and before
    c_a."""
    rng = np.random.default_rng(40 + d)
    K, n = 200, 1037
    x, ca, far = _k15_case(rng, d, K)
    fill = T.normalize(_clustered(n - 1, d, 12, d))
    g_row = gram_hw(eng, x[None], far)[0]
    g_fill = gram_hw(eng, fill, far)
    e_fill = T.exact_d2_table(fill, far)
    j = int(np.argmax(ca))                                              # a positive coordinate: bits grow with the value
    lo_bits = int(ca.view(np.int32)[j])
    hi_bits = int(np.float32(ca[j] + 0.2).view(np.int32))
    nx = P.nrm2(x[None])
    for ia, ib in ((5, 9), (5, 150), (140, 3)):
        cen = far.copy()
        cen[ia] = ca
        gr = g_row.copy()
        gr[ia] = gram_hw(eng, x[None], ca[None])[0, 0]
        gf = g_fill.copy()
        gf[:, ia] = gram_hw(eng, fill, ca[None])[:, 0]
        ef = e_fill.copy()
        ef[:, ia] = T.exact_d2_table(fill, ca[None])[:, 0]

        def centres(bits):
            c = cen.copy()
            c[ib] = _with_bits(ca, j, bits)
            return c

        def dec(bits):
            c = centres(bits)
            g = gr.copy()
            g[ib] = gram_hw(eng, x[None], c[ib:ib + 1])[0, 0]
            ok, c1 = T.assign_decide(d, nx, P.nrm2(c), g[None])
            return (bool(ok[0]), int(c1[0]) if ok[0] else -1)

        assert dec(lo_bits) == (False, -1)                              # c_b = c_a: a tie
        assert dec(hi_bits) == (True, ia)
        p0, p1 = _edge(dec, lo_bits, hi_bits)
        assert {dec(p0)[0], dec(p1)[0]} == {False, True}
        for bits in (p0, p1):
            c = centres(bits)
            cn = P.nrm2(c)
            g = gr.copy()
            g[ib] = gram_hw(eng, x[None], c[ib:ib + 1])[0, 0]
            ok, _ = T.assign_decide(d, nx, cn, g[None])
            want_x = int(T.exact_argmin(x[None], c)[0])
            labels, _, rech = eng.kmeans_assign(_cuda(x[None]), _cuda(c))
            assert rech == int(not ok[0]) and labels.item() == want_x, (ia, ib, bits)
            gfb = gf.copy()
            gfb[:, ib] = gram_hw(eng, fill, c[ib:ib + 1])[:, 0]
            efb = ef.copy()
            efb[:, ib] = T.exact_d2_table(fill, c[ib:ib + 1])[:, 0]
            ok_f, _ = T.assign_decide(d, P.nrm2(fill), cn, gfb)
            want_f = np.argmin(efb, axis=1)
            for pos in (0, 127, 128, n - 1):
                pool = np.insert(fill, pos, x, axis=0)
                labels, _, rech = eng.kmeans_assign(_cuda(pool), _cuda(c))
                assert rech == int((~ok_f).sum()) + int(not ok[0]), (ia, ib, bits, pos)
                assert labels.cpu().numpy().tolist() == np.insert(want_f, pos, want_x).tolist()


# ---- C. K18's fallback count predicted row by row ----------------------------------------------------------------------
def _fallbacks(d, x, y, G, k):
    """K18's fallback decision per row from the fp32 dot products G [n, m]: one decision per row (asserted)."""
    L = CO.screen_lower(d, P.nrm2(x)[:, None], P.nrm2(y)[None, :], G)
    dec = CO.fallback_decide(L, lambda r, c: P.exact_d2(x[r], y[c]), k)
    assert all(len(s) == 1 for s in dec)
    return np.array([next(iter(s)) for s in dec])


@pytest.mark.parametrize("m", [32, 33, 129, 700])
@pytest.mark.parametrize("d", [28, 64, 520, 2048])
def test_k18_falls_back_on_the_rows_its_band_predicts(eng, d, m):
    """Clustered rows of mixed norms with duplicated and one-ulp references: K18's fallback count equals the count
    fallback_decide gives from K3's g, for k = 1, 10, 32 (none at m <= 32), and the result is the oracle's bit for bit."""
    n = 1037
    x, y = _rows(n, m, d, 17 * d + m)
    G = gram_hw(eng, x, y)
    xt, yt = _cuda(x), _cuda(y)
    for k in (1, 10, 32):
        pred = _fallbacks(d, x, y, G, k)
        idx, d2, fb = eng.knn(xt, yt, k)
        assert fb == int(pred.sum()), (d, m, k, fb, int(pred.sum()))
        if m <= 32:
            assert fb == 0
        want_i, want_d = CO.knn(x, y, k)
        assert idx.cpu().numpy().tolist() == want_i.tolist()
        assert (d2.cpu().numpy().view(np.uint64) == want_d.view(np.uint64)).all()


# ---- D. K18 at its decision edge, to one ulp ---------------------------------------------------------------------------
def _k18_refs(rng, d, k, m, iv):
    """(x, Y, coordinate j, lo / hi bit patterns of Y[iv, j]) for a row x whose decision turns on reference iv.
    k = 32: 32 references along a ray from x and iv on the same ray, starting on the 32nd (L* < E_32: a fallback) and
    moving outwards.  k = 1: the nearest reference y0 and 31 near-copies one to three ulps away in one coordinate (inside
    its band); iv starts on y0 and moves away.  Far references (near -x) fill the columns up to m."""
    x = (2.0 * _unit(rng, 1, d)[0]).astype(np.float32)
    u = _unit(rng, 1, d)[0].astype(np.float64)
    Y = (-x[None] + 0.3 * _unit(rng, m, d)).astype(np.float32)
    others = [c for c in range(m) if c != iv][:32]
    if k == 32:
        for q, c in enumerate(others):
            Y[c] = (x + (0.3 + 0.01 * q) * u).astype(np.float32)
        start = Y[others[-1]]
    else:
        y0 = (x + 0.3 * u).astype(np.float32)
        for q, c in enumerate(others):
            Y[c] = y0
            if q:
                jj = (q * 7) % d
                Y[c, jj] = np.nextafter(np.nextafter(y0[jj], np.float32(np.inf)), np.float32(np.inf)) if q % 2 else \
                    np.nextafter(y0[jj], np.float32(-np.inf))
        start = y0
    j = int(np.argmax(np.where(start > 0, u, -np.inf)))                # start_j > 0 and u_j > 0: up is away from x
    assert start[j] > 0 and u[j] > 0
    Y[iv] = start
    lo = int(start.view(np.int32)[j])
    hi = int(np.float32(start[j] + 0.3).view(np.int32))
    return x, Y, j, lo, hi


@pytest.mark.parametrize("iv,m", [(0, 33), (150, 200)])
@pytest.mark.parametrize("k", [1, 32])
def test_k18_decides_at_its_fallback_edge(eng, k, iv, m):
    """Reference iv bisected over the fp32 bit patterns of one coordinate until L* crosses E_k (fallback_decide on K3's
    g); at both patterns K18 on the row alone falls back (or not) as predicted and inside a 1037-row pool the count is
    the prediction, with idx / d2 the oracle's bit for bit.  iv = 0 is offered first and evicted; iv = 150 sits in a
    later column tile."""
    d, n = 64, 1037
    rng = np.random.default_rng(50 + k + iv)
    x, Y, j, lo_bits, hi_bits = _k18_refs(rng, d, k, m, iv)
    fill = _rows(n - 1, m, d, 60 + k)[0]
    g_row = gram_hw(eng, x[None], Y)[0]
    g_fill = gram_hw(eng, fill, Y)

    def refs(bits):
        out = Y.copy()
        out[iv] = _with_bits(Y[iv], j, bits)
        return out

    def dec(bits):
        y = refs(bits)
        g = g_row.copy()
        g[iv] = gram_hw(eng, x[None], y[iv:iv + 1])[0, 0]
        return bool(_fallbacks(d, x[None], y, g[None], k)[0])

    assert dec(lo_bits) and not dec(hi_bits)
    p0, p1 = _edge(dec, lo_bits, hi_bits)
    for bits in (p0, p1):
        y = refs(bits)
        want = dec(bits)
        idx, d2, fb = eng.knn(_cuda(x[None]), _cuda(y), k)
        want_i, want_d = CO.knn(x[None], y, k)
        assert fb == int(want), (k, iv, bits)
        assert idx.cpu().numpy().tolist() == want_i.tolist()
        assert (d2.cpu().numpy().view(np.uint64) == want_d.view(np.uint64)).all()
        gf = g_fill.copy()
        gf[:, iv] = gram_hw(eng, fill, y[iv:iv + 1])[:, 0]
        pred_fill = int(_fallbacks(d, fill, y, gf, k).sum())
        pool = np.insert(fill, 700, x, axis=0)
        idx, d2, fb = eng.knn(_cuda(pool), _cuda(y), k)
        want_i, want_d = CO.knn(pool, y, k)
        assert fb == pred_fill + int(want), (k, iv, bits)
        assert idx.cpu().numpy().tolist() == want_i.tolist()
        assert (d2.cpu().numpy().view(np.uint64) == want_d.view(np.uint64)).all()


# ---- E. K18's band on the hardware across its whole norm range ---------------------------------------------------------
@pytest.mark.parametrize("s", [-60, 48])
@pytest.mark.parametrize("d", [64, 2048])
def test_probe_is_exact_at_the_ends_of_k18s_norm_range(eng, d, s):
    rng = np.random.default_rng(d + s)
    a = rng.integers(-8, 9, size=(200, d)).astype(np.float32)
    b = rng.integers(-8, 9, size=(12, d)).astype(np.float32)
    G = gram_hw(eng, np.ldexp(a, s), np.ldexp(b, s))
    assert (G.astype(np.float64) == np.ldexp(a.astype(np.float64) @ b.astype(np.float64).T, 2 * s)).all()


SCALES = (-60, -20, 0, 20, 49)


def _scaled_families(rng, d):
    """The bound families at each scale 2^s, plus rows with fp32-subnormal entries (all of them, or all but a spike) and
    a zero row: (rows, scale name per row, family per row)."""
    fam = P.bound_families(rng, d)
    names = np.concatenate([[f] * len(v) for f, v in fam.items()])
    base = np.concatenate(list(fam.values()))
    rows, sc, fa = [], [], []
    for s in SCALES:
        rows.append(np.ldexp(base, s).astype(np.float32))
        sc += [f"2^{s}"] * len(base)
        fa += list(names)
    sub = np.ldexp(rng.normal(size=(3, d)), -135).astype(np.float32)    # |entries| ~ 2^-135 < 2^-126
    spike = sub.copy()
    spike[:, 0] = np.float32(2.0 ** -60)
    extra = np.concatenate([sub, spike, np.zeros((1, d), dtype=np.float32)])
    assert (np.abs(sub) < 2.0 ** -126).all() and (sub != 0).any()
    rows.append(extra)
    sc += ["subnormal"] * len(extra)
    fa += ["subnormal"] * 3 + ["spike_over_subnormal"] * 3 + ["zero"]
    return np.concatenate(rows), np.array(sc), np.array(fa)


@pytest.mark.parametrize("d", [64, 2048])
def test_k18_band_holds_across_the_norm_range_on_the_h100(eng, d):
    """|d2~_hw - exact_d2| <= CO.band for every ordered pair of the bound families rescaled by 2^s, s in SCALES, mixed
    scales included, and of rows with fp32-subnormal entries; prints the worst err / b per scale and family."""
    rng = np.random.default_rng(70 + d)
    X, sc, fa = _scaled_families(rng, d)
    n2 = P.nrm2(X)
    assert n2.max() <= 2.0 ** 100
    G = gram_hw(eng, X)
    E = T.exact_d2_table(X, X)
    d2 = CO.screen_d2(n2[:, None], n2[None, :], G)
    R = np.abs(d2 - E) / CO.band(d, n2[:, None], n2[None, :])
    worst = {}
    for key, lab in (("scale", sc), ("family", fa)):
        worst[key] = {v: float(max(R[lab == v].max(), R[:, lab == v].max())) for v in dict.fromkeys(lab)}
    a, b = np.unravel_index(np.argmax(R), R.shape)
    print(f"\nH100 K18 band d={d}: worst err/b {R.max():.4f} ({sc[a]} {fa[a]} x {sc[b]} {fa[b]}); by scale: "
          + ", ".join(f"{v} {w:.4f}" for v, w in worst["scale"].items()) + "; by family: "
          + ", ".join(f"{v} {w:.4f}" for v, w in worst["family"].items()))
    assert R.max() <= 1.0, f"d={d}: err/b = {R.max():.4f} at rows {a}, {b}"


def test_k18_accepts_nrm2_up_to_2_100_and_refuses_one_ulp_more(eng):
    from active_learning_b200._lib import AlqError
    rng = np.random.default_rng(80)
    x = rng.normal(size=(50, 64)).astype(np.float32)
    y = rng.normal(size=(40, 64)).astype(np.float32)
    y[3] = 0.0
    y[3, 5] = np.float32(2.0 ** 50)                                     # nrm2 = 2^100 exactly
    x[7] = y[3]
    assert P.nrm2(y[3:4])[0] == 2.0 ** 100
    for k in (1, 10):
        idx, d2, _ = eng.knn(_cuda(x), _cuda(y), k)
        want_i, want_d = CO.knn(x, y, k)
        assert idx.cpu().numpy().tolist() == want_i.tolist()
        assert (d2.cpu().numpy().view(np.uint64) == want_d.view(np.uint64)).all()
    y[3, 5] = np.nextafter(np.float32(2.0 ** 50), np.float32(np.inf))
    with pytest.raises(AlqError, match=r"1 rows have a squared norm that is not finite or exceeds 2\^100"):
        eng.knn(_cuda(x[:6]), _cuda(y), 3)
    idx, _, _ = eng.knn(_cuda(x[:6]), _cuda(y[4:]), 3)
    assert idx.cpu().numpy().tolist() == CO.knn(x[:6], y[4:], 3)[0].tolist()


# ---- F. K15's domain ---------------------------------------------------------------------------------------------------
def test_k15_refuses_norms_outside_its_domain(eng):
    """The zero row against two centres of |c|^2 ~ 6e7 (a permutation of each other), where the band would certify
    centre 1 and the exact argmin is 0, is refused by name with the labels untouched; so are rows of squared norm 4,
    NaN centres, and Engine.kmeans on unnormalised rows.  Zero rows and rows pushed to nrm2 = 2 against centres inside
    the unit ball are accepted and get the exact argmin, and the context stays usable."""
    from active_learning_b200._lib import AlqError
    x, cen = k15_counterexample()
    assert T.exact_argmin(x, cen)[0] == 0
    labels = torch.full((1,), 7, dtype=torch.int32, device="cuda")
    with pytest.raises(AlqError, match=r"2 rows or centres have a squared norm that is not in \[0, 2\]"):
        eng.kmeans_assign(_cuda(x), _cuda(cen), labels)
    assert labels.item() == 7
    rng = np.random.default_rng(90)
    xhat = T.normalize(_clustered(600, 64, 8, 90))
    cen = _centres(rng, xhat, 20)
    with pytest.raises(AlqError, match=r"600 rows or centres have a squared norm that is not in \[0, 2\]"):
        eng.kmeans_assign(_cuda(2 * xhat), _cuda(cen))
    bad = cen.copy()
    bad[4, 2] = np.nan
    with pytest.raises(AlqError, match=r"1 rows or centres"):
        eng.kmeans_assign(_cuda(xhat), _cuda(bad))
    with pytest.raises(AlqError, match=r"rows or centres have a squared norm that is not in \[0, 2\]"):
        eng.kmeans(_cuda(3 * xhat), 0, rng.random(9), 10)
    z = xhat.copy()
    z[::3] = 0.0                                                        # zero rows
    z[1::3] = (z[1::3].astype(np.float64) * np.sqrt(2.0) * (1 - 2.0 ** -20)).astype(np.float32)
    assert P.nrm2(z).max() <= 2.0
    labels, changed, _ = eng.kmeans_assign(_cuda(z), _cuda(cen))
    assert labels.cpu().numpy().tolist() == T.exact_argmin(z, cen).tolist() and changed == len(z)
    got, _, it, _ = eng.kmeans(_cuda(xhat), 0, rng.random(9), 10)
    assert it >= 1 and got.shape[0] == len(xhat)
