"""The 3xTF32 bound of DESIGN section 4 measured on the H100's own tensor cores, K13's rechecks predicted pair by pair,
and K14 at its segment limit.

K3 (alq_mindist_tc.cu) and K13 (alq_probcover.cu) issue the same wgmma chain, tc::ring_mma of alq_wgmma.cuh: the same
split_tf32, per 8-wide k-step hi hi', hi lo', lo hi', k ascending, into one m64n128 fp32 fragment.  With zero norms and
one column row, K3 returns fl(fl(0 + 0) - 2 acc) = -2 g exactly, so g_hw(X, y) = -0.5 K3(X, 0, y, 0) reads the tensor
core's fp32 dot product g of any operand pair through the public API.  The probe is established first (exact where it must be, on the tensor path,
independent of the pair's place in the tile); then it holds E against fp64 truth and predicts K13's band decisions.
"""
import contextlib
import ctypes as C

import numpy as np
import pytest
import torch

import probcover_oracle as P

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from active_learning_b200.engine import Engine
    return Engine()


@contextlib.contextmanager
def _k3_impl(eng, impl):
    eng.set_option("k3_impl", impl)
    try:
        yield
    finally:
        eng.set_option("k3_impl", 0)


def _dev(x):
    """fp32 rows on the device, zero columns up to K3's tensor-path minimum of 32 (K13's TMA zero-fills the same
    columns, so the chain is the same single k-block)."""
    x = np.asarray(x, dtype=np.float32)
    if x.shape[1] < 32:
        x = np.concatenate([x, np.zeros((x.shape[0], 32 - x.shape[1]), dtype=np.float32)], axis=1)
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _k3(eng, X, Y, impl=2, reduce_max=False):
    """K3 with zero norms: min_j (max_j) of -2 g(X_i, Y_j), as fp32 [n] on the host."""
    zx = torch.zeros(X.shape[0], dtype=torch.float32, device="cuda")
    zy = torch.zeros(Y.shape[0], dtype=torch.float32, device="cuda")
    with _k3_impl(eng, impl):
        out = eng.min_dist(X, zx, Y, zy, reduce_max=reduce_max)
    return out.cpu().numpy()


def gram_hw(eng, a, b=None, impl=2):
    """G[i, j] = g(a_i, b_j) with a_i the row operand and b_j the column operand: one K3 call per column."""
    A = _dev(a)
    B = A if b is None else _dev(b)
    zx = torch.zeros(A.shape[0], dtype=torch.float32, device="cuda")
    zy = torch.zeros(1, dtype=torch.float32, device="cuda")
    with _k3_impl(eng, impl):
        cols = [eng.min_dist(A, zx, B[j:j + 1], zy) for j in range(B.shape[0])]
    return (torch.stack(cols, dim=1) * -0.5).cpu().numpy()


def _families(d):
    fam = P.bound_families(np.random.default_rng(100 + d), d)       # the rows test_probcover.py emulates
    names = np.concatenate([[k] * len(v) for k, v in fam.items()])
    return names, np.concatenate(list(fam.values()))


# ---- 1. the probe -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [4, 36, 2048])
def test_probe_is_exact_on_tf32_exact_operands(eng, d):
    rng = np.random.default_rng(d)
    a = rng.integers(-8, 9, size=(200, d)).astype(np.float32)      # lo = 0, every partial sum below 2^24
    b = rng.integers(-8, 9, size=(12, d)).astype(np.float32)
    G = gram_hw(eng, a, b)
    assert (G.astype(np.float64) == a.astype(np.float64) @ b.astype(np.float64).T).all()


def test_probe_is_on_the_tensor_path(eng):
    rng = np.random.default_rng(1)
    a = P.normalize(rng.normal(size=(256, 64)).astype(np.float32))
    b = a[:16]
    tc, simt = gram_hw(eng, a, b, impl=2), gram_hw(eng, a, b, impl=1)
    assert (tc != simt).any()
    truth = a.astype(np.float64) @ b.astype(np.float64).T
    assert np.abs(tc - truth).max() <= P.screen_bound(64, 1.0, 1.0) * 1.01


@pytest.mark.parametrize("d", [36, 2048])
def test_probe_is_independent_of_the_pairs_place_in_the_tile(eng, d):
    names, xh = _families(d)
    X = _dev(np.concatenate([xh, xh[::-1]]))                           # two row tiles (and a partial one)
    for j in range(0, len(xh), 5):
        # y in all 128 rows of one column tile: every column position gives the same g, so min = max
        Y = _dev(np.repeat(xh[j:j + 1], 128, axis=0))
        lo, hi = _k3(eng, X, Y), _k3(eng, X, Y, reduce_max=True)
        assert (lo == hi).all(), (names[j], d)
        assert (lo == _k3(eng, X, Y[:1])).all()
        # one x row in all 128 rows of a row tile (both consumer warpgroups): every output equal
        Xj = _dev(np.repeat(xh[j:j + 1], 128, axis=0))
        out = _k3(eng, Xj, X[: len(xh)][::7].contiguous())
        assert (out == out[0]).all(), (names[j], d)


# ---- 2. the bound on the H100 -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [4, 28, 36, 64, 520, 2048])
def test_screen_bound_holds_on_the_h100(eng, d):
    """|g_hw - <x_i, x_j>| <= E for every ordered pair of the bound families; prints the worst err / E per family."""
    names, xh = _families(d)
    m = len(xh)
    G = gram_hw(eng, xh).astype(np.float64)
    i, j = np.triu_indices(m)
    T = np.zeros((m, m))
    T[i, j] = P.exact_dots(xh[i], xh[j])
    T[j, i] = T[i, j]
    nrm = P.nrm2(xh)
    R = np.abs(G - T) / P.screen_bound(d, nrm[:, None], nrm[None, :])
    worst = {f: float(max(R[names == f].max(), R[:, names == f].max())) for f in dict.fromkeys(names)}
    a, b = np.unravel_index(np.argmax(R), R.shape)
    print(f"\nH100 3xTF32 bound d={d}: worst err/E {R.max():.4f} ({names[a]} x {names[b]}); "
          + ", ".join(f"{f} {v:.4f}" for f, v in worst.items()))
    assert R.max() <= 1.0, f"d={d}: err/E = {R.max():.4f} at {names[a]} x {names[b]} (rows {a}, {b})"


# ---- 3. K13's recheck count predicted pair by pair ---------------------------------------------------------------------
def _k13(eng, x, delta):
    """K13's count and fill passes into buffers this test owns: (xhat, row_ptr, cols, recheck) on the host."""
    from active_learning_b200.engine import _ptr
    n, d = x.shape
    nt = (n + 127) // 128
    xhat = torch.empty((n, d), dtype=torch.float32, device="cuda")
    tile = torch.empty(n * nt, dtype=torch.int32, device="cuda")
    row_ptr = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    dh, nnz, rech = C.c_double(delta), C.c_int64(0), C.c_int64(0)
    eng._check(eng.lib.alq_probcover_graph(eng._h, _ptr(x), n, d, d, C.byref(dh), _ptr(xhat), _ptr(tile), _ptr(row_ptr),
                                           None, C.byref(nnz), C.byref(rech), eng._stream()), "alq_probcover_graph")
    cols = torch.empty(max(nnz.value, 1), dtype=torch.int32, device="cuda")
    eng._check(eng.lib.alq_probcover_graph(eng._h, None, n, d, d, C.byref(dh), _ptr(xhat), _ptr(tile), _ptr(row_ptr),
                                           _ptr(cols), C.byref(nnz), C.byref(rech), eng._stream()), "alq_probcover_graph")
    return xhat.cpu().numpy(), row_ptr.cpu().numpy(), cols[:nnz.value].cpu().numpy(), int(rech.value)


def _flip(dec, lo, hi):
    """Adjacent fp64 radii lo < hi with dec(lo) != dec(hi), by bisection from such a pair."""
    assert dec(lo) != dec(hi)
    while True:
        mid = 0.5 * (lo + hi)
        if not lo < mid < hi:
            return lo, hi
        if dec(mid) == dec(lo):
            lo = mid
        else:
            hi = mid


def _radii(d, ni, nj, g):
    """Radii that put the pair's d2 = ni + nj - 2 g inside the band (d2 = delta^2 - 0.999 b, - b / 2, + 0), just outside
    (+ 1.01 b), and on both sides of either band edge to the fp64 ulp, each with the decision it must get."""
    d2 = (ni + nj) - 2.0 * float(g)
    coef = 2.0 * P.screen_bound(d, 1.0, 1.0) * (1.0 + 1e-6)
    dec = lambda delta: int(P.screen_decide(d, ni, nj, g, delta))     # noqa: E731
    out = []
    for p in (-0.999, -0.5, 0.0, 1.01):
        delta2 = d2
        for _ in range(4):                                             # b depends on delta through the slack
            delta2 = d2 - p * (coef * np.sqrt(ni * nj) + 1e-9 * delta2 + 1e-10)
        delta = float(np.sqrt(delta2))
        out.append((delta, P.NONE if p > 1 else P.RECHECK))
    b = coef * np.sqrt(ni * nj) + 1e-9 * d2 + 1e-10
    for lo, hi in ((np.sqrt(d2 - 2 * b), np.sqrt(d2)), (np.sqrt(d2), np.sqrt(d2 + 2 * b))):
        out += [(delta, dec(delta)) for delta in _flip(dec, float(lo), float(hi))]
    for delta, want in out:
        assert dec(delta) == want
    return out


def _targets(rng, xhat, G, n2, tile):
    """Pairs whose radii the test places: an off-diagonal-tile pair with g(i, j) != g(j, i) (the order of hi lo' and
    lo hi' shows), a pair of the last tile with an earlier one, and a pair inside a diagonal tile.  Rows that occur twice
    are left out: a mirrored copy of the pair would flip the other way and hide a wrong order in the count."""
    _, inv, cnt = np.unique(xhat, axis=0, return_inverse=True, return_counts=True)
    single = cnt[inv.ravel()] == 1
    d2 = n2[:, None] + n2[None, :] - 2.0 * G
    ok = (d2 > 0.05) & (d2 < 3.9) & single[:, None] & single[None, :]
    off = ok & (tile[:, None] < tile[None, :])
    asym = off & (G != G.T)
    picks = []
    for cand in (asym if asym.any() else off, off & (tile[None, :] == tile[-1]),
                 ok & (tile[:, None] == tile[None, :]) & ~np.eye(len(tile), dtype=bool)):
        i, j = np.nonzero(cand)
        k = rng.integers(len(i))
        picks.append((int(i[k]), int(j[k])))
    return picks, bool(asym.any())


@pytest.mark.parametrize("n", [300, 640])
@pytest.mark.parametrize("d", [28, 64, 520, 2048])
def test_k13_rechecks_the_pairs_its_band_predicts(eng, n, d):
    """At radii placed in and at the edges of chosen pairs' bands: K13's x̂ is P.normalize's, its recheck count equals the
    count screen_decide gives from K3's g pair by pair, and its CSR is P.graph's.  A band-edge pair flips on one ulp of
    K13's g, so this holds K13's MMA chain to K3's bit for bit and its band to DESIGN section 4's formula."""
    rng = np.random.default_rng(7 * n + d)
    _, fam = _families(d)
    x = rng.normal(size=(n, d)).astype(np.float32)
    x[rng.choice(n, len(fam), replace=False)] = fam
    xt = torch.from_numpy(x).cuda()
    xhat = P.normalize(x)
    G = gram_hw(eng, xhat)
    n2 = P.nrm2(xhat)
    tile = np.arange(n) // 128
    decided = tile[:, None] <= tile[None, :]      # K13's tile (tile i, tile j); a diagonal tile decides both orders
    targets, asym = _targets(rng, xhat, G, n2, tile)
    assert asym or d == 28, "no pair with g(i, j) != g(j, i) off the diagonal tiles"
    for i, j in targets:
        for delta, want in _radii(d, n2[i], n2[j], G[i, j]):
            got_xhat, rp, cl, rech = _k13(eng, xt, delta)
            assert np.array_equal(got_xhat.view(np.uint32), xhat.view(np.uint32))
            pred = int((P.screen_decide(d, n2[:, None], n2[None, :], G, delta) == P.RECHECK)[decided].sum())
            assert rech == pred, (f"n={n} d={d} pair ({i}, {j}) tiles ({tile[i]}, {tile[j]}) delta={delta!r} "
                                  f"(pair decision {want}): K13 rechecked {rech}, the band predicts {pred}")
            want_rp, want_cl = P.graph(xhat, delta)
            assert rp.tolist() == want_rp.tolist() and cl.tolist() == want_cl.tolist()


# ---- 4. K14 at its limits ----------------------------------------------------------------------------------------------
def _csr(n, pairs):
    adj = [{r} for r in range(n)]
    for a, b in pairs:
        adj[a].add(b)
        adj[b].add(a)
    row_ptr = np.zeros(n + 1, dtype=np.int64)
    row_ptr[1:] = np.cumsum([len(s) for s in adj])
    return row_ptr, np.concatenate([sorted(s) for s in adj]).astype(np.int32)


def test_k14_at_the_65535_row_segment_limit(eng):
    """n = 65 535 G rows over G = SMs CTAs: every segment holds 65 535 rows, the largest row offset a key word carries is
    0xfffe (next to the empty marker 0xffff).  On the identity graph every degree is 1, so the picks are the unlabeled
    rows in ascending order.  One row more is refused by name, and the context stays usable."""
    from active_learning_b200._lib import AlqError
    G = torch.cuda.get_device_properties(eng.device).multi_processor_count
    seg = 65535
    n = seg * G
    assert min(G, -(-n // 256)) == G
    free = sorted({b * seg + off for b, off in [(0, 0xfffe), (1, 0xfffe), (G // 2, 0xfffe), (G - 1, 0xfffe),
                                                 (0, 0), (1, 0), (G - 1, 0), (G // 3, 0x8000)]})
    row_ptr = torch.arange(n + 1, dtype=torch.int64, device="cuda")
    cols = torch.arange(n, dtype=torch.int32, device="cuda")
    lab = torch.ones(n, dtype=torch.uint8, device="cuda")
    lab[torch.tensor(free, device="cuda")] = 0
    picks, steps = eng.probcover_select(row_ptr, cols, lab, len(free) + 7)
    assert steps == len(free) and picks.tolist() == free
    del row_ptr, cols, lab
    row_ptr = torch.arange(n + 2, dtype=torch.int64, device="cuda")
    cols = torch.arange(n + 1, dtype=torch.int32, device="cuda")
    lab = torch.zeros(n + 1, dtype=torch.uint8, device="cuda")
    with pytest.raises(AlqError, match=r"65535 rows per CTA segment"):
        eng.probcover_select(row_ptr, cols, lab, 1)
    del row_ptr, cols, lab
    rp, cl = _csr(5, [(0, 1), (3, 4), (2, 4)])
    picks, steps = eng.probcover_select(torch.from_numpy(rp).cuda(), torch.from_numpy(cl).cuda(),
                                        torch.zeros(5, dtype=torch.uint8, device="cuda"), 5)
    assert picks.tolist() == P.greedy(rp, cl, np.zeros(5, dtype=bool), 5).tolist() == [4, 0] and steps == 2


@pytest.mark.parametrize("n", [1, 2, 256, 257])
def test_k14_small_pools_equal_the_oracle(eng, n):
    """One CTA up to 256 rows, two from 257: hand-written graphs with degree ties inside and across the segments."""
    rng = np.random.default_rng(n)
    graphs = [[]]
    if n >= 2:
        graphs.append([(0, n - 1)])
    if n >= 256:
        ring = [(r, (r + 1) % n) for r in range(n)]
        hubs = [(h, h + k) for h in (5, 131, 200) for k in range(1, 9)]       # three equal balls; 131 and 200 in segment 1
        graphs += [ring, ring + hubs, [tuple(p) for p in rng.integers(0, n, size=(3 * n, 2))]]
    for pairs in graphs:
        rp, cl = _csr(n, pairs)
        for lab in (np.zeros(n, dtype=bool), rng.random(n) < 0.1):
            for budget in sorted({1, min(3, n), n}):
                want = P.greedy(rp, cl, lab, budget)
                picks, steps = eng.probcover_select(torch.from_numpy(rp).cuda(), torch.from_numpy(cl).cuda(),
                                                    torch.from_numpy(lab.astype(np.uint8)).cuda(), budget)
                assert picks.tolist() == want.tolist() and steps == len(want), (n, len(pairs), budget)
