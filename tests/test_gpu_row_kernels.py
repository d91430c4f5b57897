"""The streaming row kernels (K1 scores, K2 BADGE factors, K2p, row norms, K6 MASE margins), the top-B selection (K1b)
and the fused K1 + K1b tail on every dispatch route and register width, against the float64 restatement in
tests/row_reference.py with per-row error bounds derived from the kernels' arithmetic.

Dispatch (alq_score.cu: alq_score_softmax, alq_badge_factors; alq_mase.cu: alq_mase_margins):
  vec      = c % 4 == 0, ld % 4 == 0, 16-byte aligned base (K2: also lda), c <= 2048 (K6: c <= 1024, ldr == c)
  pipe     = vec and ld == c and n >= 4096          -> rows_pipe_kernel<NV, mode>   (bulk-copy tile ring, R rows a tile)
  direct   = vec otherwise                          -> score_rows_vec / badge_factors_vec / mase_rows_{min,vec}<NV>
  generic  = everything else                        -> score_rows_generic / badge_factors_generic / mase_rows_generic
  NV = ceil(c / 128) rounded up to {1, 2, 4, 8, 16} (K6: c <= 1024, so NV <= 8).
Inputs per width (test_route_width_matrix): the same [4097, c] logits as
  direct       contiguous, n = 4095                  (c % 4 != 0 or c > 2048: generic)
  direct_ld    [4096, c + 4] slab sliced to c columns (ld != c)
  pipe_4096    contiguous, n = 4096                  (a multiple of every tile height R)
  pipe_4097    contiguous, n = 4097                  (not a multiple of R = min(32, 16384 // (4 c)) for any width here)
  misaligned   slab[:, 1:c + 1] of a [4097, c + 8] slab: base 4 bytes off 16 -> generic
(route, NV) pairs reached, c <= 4096:
  K1 (3 modes), K2: direct and pipe with NV 1 (c = 4, 64, 128), 2 (132, 256), 4 (260, 512), 8 (516, 1000, 1024),
                    16 (1028, 2048); generic at every width (misaligned) and for c = 37, 1001, 2052, 4096 on all routes.
  K6 (min-only with gmin, full radius): direct and pipe with NV 1, 2, 4, 8 (c <= 1024), generic as above for c <= 1024
                    and c = 37, 1001.
The first rows of every input are the special rows of test_row_reference.special_rows (masked classes, one finite logit,
all -inf, NaN, +inf, +-3e38, gaps below -87, ties at the maximum).  The worst err / bound per kernel is printed at the
end of the module."""
import json

import numpy as np
import pytest
import torch

import row_reference as R
from oracle import al_oracle as O
from test_row_reference import special_rows

pytestmark = pytest.mark.gpu

WIDTHS = [4, 64, 128, 132, 256, 260, 512, 516, 1000, 1024, 1028, 2048, 2052, 4096, 37, 1001]
MODES = (O.MODE_MARGIN, O.MODE_LEAST_CONFIDENCE, O.MODE_ENTROPY)
MODE_NAMES = {0: "K1 margin", 1: "K1 least confidence", 2: "K1 entropy"}
N_ROWS = 4097
WORST = {}


@pytest.fixture(scope="module")
def eng():
    from active_learning_b200.engine import Engine
    yield Engine()
    print("\nworst err / bound per kernel: " + json.dumps({k: round(v, 4) for k, v in sorted(WORST.items())}))


def vec_ok(c, cmax=2048):
    return c % 4 == 0 and c <= cmax


def check_within(name, got, ref, bound):
    """NaN exactly where the reference is NaN, infinities equal, |got - ref| <= bound elsewhere; records err / bound."""
    got = np.asarray(got, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    bound = np.broadcast_to(np.asarray(bound, dtype=np.float64), ref.shape)
    assert np.array_equal(np.isnan(got), np.isnan(ref)), name
    inf = np.isinf(ref)
    assert np.array_equal(got[inf], ref[inf]), name
    fin = np.isfinite(ref)
    err, b = np.abs(got[fin] - ref[fin]), bound[fin]
    bad = err > b
    assert not bad.any(), (name, got[fin][bad][:4], ref[fin][bad][:4], b[bad][:4])
    if err.size:
        r = float(np.max(np.where(b > 0, err / np.where(b > 0, b, 1.0), 0.0)))
        WORST[name] = max(WORST.get(name, 0.0), r)


def bits(t):
    return t.contiguous().view(torch.int32)


def logits_with_special_rows(c, seed, n=N_ROWS):
    rng = np.random.default_rng(seed)
    z = (rng.standard_normal((n, c)) * 3).astype(np.float32)
    sp = special_rows(c, rng)
    z[:len(sp)] = sp
    z[len(sp)::97] *= 20.0                       # some rows at a high temperature: tiny probabilities
    return z


def sample_rows(n, seed, k=256):
    rng = np.random.default_rng(seed)
    return np.unique(np.concatenate([np.arange(12), rng.choice(n, k, replace=False), [n - 2, n - 1]]))


def routes(z):
    """(name, tensor, n) of every route input built from the same logits (see the module docstring)."""
    n, c = z.shape
    dev = torch.from_numpy(z).cuda()
    ld = torch.full((n - 1, c + 4), float("nan"), device="cuda")
    ld[:, :c] = dev[:n - 1]
    mis = torch.full((n, c + 8), float("nan"), device="cuda")
    mis[:, 1:c + 1] = dev
    out = [("direct", dev[:n - 2], n - 2), ("direct_ld", ld[:, :c], n - 1), ("pipe_4096", dev[:n - 1], n - 1),
           ("pipe_4097", dev, n), ("misaligned", mis[:, 1:c + 1], n)]
    assert out[1][1].stride(0) == c + 4 and out[4][1].data_ptr() % 16 == 4
    return out


def route_kind(name, c, cmax=2048):
    return "generic" if name == "misaligned" or not vec_ok(c, cmax) else "vec"


@pytest.mark.parametrize("c", WIDTHS)
def test_route_width_matrix(eng, c):
    """K1 (3 modes), K2 and K6 (min-only and full) on every route at this width: within the fp64 bound on a seeded row
    subsample (the special rows included), NaN exactly where the reference is NaN; routes that run the same row code
    (direct, direct_ld, pipe_*; or every route when the width only has the generic kernel) bit-identical on all rows;
    K6's pred and inf pattern equal to mase64's and its min-only minimum bit-identical to the full one."""
    z = logits_with_special_rows(c, c)
    rows = sample_rows(N_ROWS, c + 1)
    zs = z[rows]
    rts = routes(z)
    same_code = [r for r in rts if route_kind(r[0], c) == "vec"] if vec_ok(c) else rts
    # ---- K1 ----
    for mode in MODES:
        ref = R.softmax_scores64(zs, mode)
        res = {}
        for name, t, n in rts:
            res[name] = eng.score_softmax(t, mode)
            m = rows < n
            check_within(MODE_NAMES[mode], res[name].cpu().numpy()[rows[m]], ref[m],
                         R.score_bound(zs[m], mode, route_kind(name, c)))
        base = res[same_code[0][0]]
        for name, _, n in same_code[1:]:
            k = min(n, base.numel())
            assert torch.equal(bits(res[name][:k]), bits(base[:k])), (mode, name)
    # ---- K2 (bs = 128: the routes' n differ, so the last loader batch does too) ----
    a1, _ = R.badge_factors64(zs, 1)
    e1, en1 = R.badge_bound(zs, 1, "vec")
    g1, gn1 = R.badge_bound(zs, 1, "generic")
    res = {}
    for name, t, n in rts:
        a, an = eng.badge_factors(t, 128)
        res[name] = (a, an)
        m = rows < n
        bsz = R.batch_sizes(n, 128)[rows[m]][:, None]
        eb, enb = (e1, en1) if route_kind(name, c) == "vec" else (g1, gn1)
        a_h = a.cpu().numpy()
        check_within("K2 factors", a_h[rows[m], :c], a1[m] / bsz, eb[m] / bsz)
        check_within("K2 norm2", an.cpu().numpy()[rows[m]], (a1[m] ** 2).sum(1) / bsz[:, 0] ** 2, enb[m] / bsz[:, 0] ** 2)
        assert (a_h[:, c:] == 0).all()
    if vec_ok(c):
        for x, y in zip(res["direct_ld"], res["pipe_4096"]):
            assert torch.equal(bits(x), bits(y))
    # ---- K6 ----
    if c > 1024 and c not in (37, 1001):
        return
    w = np.random.default_rng(c + 2).standard_normal((c, 48)) * 0.3
    gap = eng.class_gap_inv(torch.from_numpy(w).float().cuda())
    mm64, pred64, r64 = R.mase64(zs, w.astype(np.float32))
    vec6 = vec_ok(c, 1024)
    same6 = [r for r in rts if route_kind(r[0], c, 1024) == "vec"] if vec6 else rts
    res = {}
    for name, t, n in rts:
        full, pred, radius = eng.mase_margins(t, gap, want_per_class=True)
        mn, pred2, _ = eng.mase_margins(t, gap, want_per_class=False)
        assert torch.equal(bits(mn), bits(full)) and torch.equal(pred, pred2), name
        res[name] = (full, pred, radius)
        m = rows < n
        assert np.array_equal(pred.cpu().numpy()[rows[m]], pred64[m]), name
        rad = radius.cpu().numpy()[rows[m]]
        assert np.array_equal(np.isinf(rad), np.isinf(r64[m])), name
        check_within("K6 radius", rad, r64[m], R.mase_bound(r64[m], 48))
        check_within("K6 min margin", full.cpu().numpy()[rows[m]], mm64[m], R.mase_bound(mm64[m], 48))
    base = res[same6[0][0]]
    for name, _, n in same6[1:]:
        k = min(n, base[0].numel())
        for x, y in zip(res[name], base):
            assert torch.equal(bits(x[:k]), bits(y[:k])), name


@pytest.mark.parametrize("n,c", [(1000, 1000), (5000, 1000), (5000, 132), (300, 37), (4100, 2048)])
def test_masking_a_class_leaves_the_other_rows_unchanged(eng, n, c):
    """Entropy with masked classes (-inf logits): 0 log 0 = 0.  Masking a class in every other row leaves the other rows'
    scores bit-identical, and the masked rows' entropy is finite and within the bound of the fp64 reference (before the
    fix it was NaN on every route)."""
    rng = np.random.default_rng(n + c)
    z = (rng.standard_normal((n, c)) * 3).astype(np.float32)
    zm = z.copy()
    zm[::2, rng.choice(c, max(1, c // 5), replace=False)] = -np.inf
    for mode in MODES:
        plain = eng.score_softmax(torch.from_numpy(z).cuda(), mode)
        masked = eng.score_softmax(torch.from_numpy(zm).cuda(), mode)
        assert torch.equal(bits(plain[1::2]), bits(masked[1::2]))
        route = "vec" if vec_ok(c) else "generic"
        check_within(MODE_NAMES[mode], masked.cpu().numpy()[::2], R.softmax_scores64(zm[::2], mode),
                     R.score_bound(zm[::2], mode, route))
        assert torch.isfinite(masked).all()


def special_scores(n, seed):
    """Tie-heavy scores mixed with NaN, -NaN (0xffc00000), +-inf and +-0."""
    rng = np.random.default_rng(seed)
    s = (rng.integers(0, 40, n) / 16.0 - 1.0).astype(np.float32)
    u = s.view(np.uint32)
    idx = rng.permutation(n)
    k = max(1, n // 50)
    for j, pattern in enumerate((0x7fc00000, 0xffc00000, 0x7f800000, 0xff800000, 0x00000000, 0x80000000)):
        u[idx[j * k:(j + 1) * k]] = pattern
    return s


def straddling_budgets(s):
    """Budgets that cut a tie group (the +-0 group, a finite group, +inf), land on, before and after the first NaN, plus
    1 and n."""
    order = torch.sort(torch.from_numpy(s), stable=True).values.numpy()
    n = len(s)
    first_nan = int(np.isnan(order).argmax())
    zero = int(np.flatnonzero(order == 0)[0])
    grp = int(np.flatnonzero(order == np.float32(0.5))[0])
    inf = int(np.flatnonzero(order == np.inf)[0])
    return sorted({1, zero + 2, grp + 3, inf + 1, first_nan - 1, first_nan, first_nan + 1, n})


@pytest.mark.parametrize("n", [5000, 100003])
def test_select_orders_special_scores_like_torch_stable_sort(eng, n):
    """K1b (both implementations; the cluster-resident one takes b <= 16384) and the multi-GPU pack + merge primitives:
    NaN and -NaN sort last, -0 ties with +0, ties by position, exactly `torch.sort(stable=True).indices[:b]`."""
    s = special_scores(n, n)
    ref = torch.sort(torch.from_numpy(s), stable=True).indices.numpy()
    dev = torch.from_numpy(s).cuda()
    bounds = [0, n // 3, n // 3 + 1234, n]
    try:
        for b in straddling_budgets(s):
            for impl in (1, 2) if b <= 16384 else (1,):
                eng.set_option("select_impl", impl)
                assert np.array_equal(eng.select_smallest(dev, b).cpu().numpy(), ref[:b]), (impl, b)
            eng.set_option("select_impl", 0)
            words = []
            for lo, hi in zip(bounds[:-1], bounds[1:]):
                loc = dev[lo:hi].contiguous()
                words.append(eng.topb_pack(loc, eng.select_smallest(loc, min(b, hi - lo)), lo, b))
            assert np.array_equal(eng.topb_merge(torch.cat(words), b).cpu().numpy(), ref[:b]), b
            assert np.array_equal(eng.topb_merge(torch.cat(words), b, list_len=b).cpu().numpy(), ref[:b]), b
    finally:
        eng.set_option("select_impl", 0)


@pytest.mark.parametrize("mode", MODES)
def test_fused_tail_with_nan_rows(eng, mode):
    """Pools whose rows hold NaN logits through the fused tail: NaN scores sort last in position order; b below, at and
    past the first NaN, on both ranking routes."""
    n, c, n_nan = 30011, 1000, 500
    g = torch.Generator(device="cuda").manual_seed(5 + mode)
    logits = torch.randn(n, c, device="cuda", generator=g) * 3
    nan_rows = torch.randperm(n, generator=g, device="cuda")[:n_nan]
    logits[nan_rows, 17] = float("nan")
    ref_s = eng.score_softmax(logits, mode)
    assert int(torch.isnan(ref_s).sum()) == n_nan
    order = torch.sort(ref_s.cpu(), stable=True).indices.numpy()
    try:
        for buckets in (1, 0):
            eng.set_option("tail_buckets", buckets)
            for b in (n - n_nan - 1, n - n_nan, n - n_nan + 1, n):
                s, p = eng.uncertainty_tail(logits, mode, b)
                eng.uncertainty_tail_timing()                      # the fused launch ran
                assert torch.equal(bits(s), bits(ref_s))
                assert np.array_equal(p.cpu().numpy(), order[:b]), (buckets, b)
    finally:
        eng.set_option("tail_buckets", 1)


@pytest.mark.parametrize("c", [132, 260, 516, 2048])
def test_fused_tail_at_every_register_width(eng, c):
    """The fused tail at NV = 2, 4, 8 and 16 (c = 2048: the spilling instantiation), b from 1 to n, against the two
    separate kernels, both ranking routes."""
    n = 30011
    g = torch.Generator(device="cuda").manual_seed(c)
    logits = torch.randn(n, c, device="cuda", generator=g) * 3
    try:
        for mode in MODES:
            ref_s = eng.score_softmax(logits, mode)
            for b in (1, 777, n // 3, n):
                ref_p = eng.select_smallest(ref_s, b)
                for buckets in (1, 0):
                    eng.set_option("tail_buckets", buckets)
                    s, p = eng.uncertainty_tail(logits, mode, b)
                    eng.uncertainty_tail_timing()
                    assert torch.equal(bits(s), bits(ref_s)) and torch.equal(p, ref_p), (mode, b, buckets)
            sub = np.random.default_rng(c).choice(n, 200, replace=False)
            zs = logits[torch.from_numpy(sub).cuda()].cpu().numpy()
            check_within(MODE_NAMES[mode], ref_s.cpu().numpy()[sub], R.softmax_scores64(zs, mode),
                         R.score_bound(zs, mode, "vec"))
    finally:
        eng.set_option("tail_buckets", 1)


def test_fused_tail_size_boundary(eng):
    """The tail fuses while 4096 <= n and 5 n <= sm_count * 2048 * 4 (the per-CTA key lists absorb any imbalance):
    fused at n = 4096 and at the limit, split at 4095 and one row past it.  The timing stamps exist only after a fused
    launch; the result is the same either way."""
    from active_learning_b200._lib import AlqError
    sm = torch.cuda.get_device_properties(eng.device).multi_processor_count
    n_max = sm * 2048 * 4 // 5
    g = torch.Generator(device="cuda").manual_seed(3)
    big = torch.randn(n_max + 1, 8, device="cuda", generator=g) * 3
    for n, fused in ((4095, False), (4096, True), (n_max, True), (n_max + 1, False)):
        logits = big[:n]
        for b in (1000, n // 2):
            ref_s = eng.score_softmax(logits, 0)
            s, p = eng.uncertainty_tail(logits, 0, b)
            if fused:
                eng.uncertainty_tail_timing()
            else:
                with pytest.raises(AlqError):
                    eng.uncertainty_tail_timing()
            assert torch.equal(bits(s), bits(ref_s)) and torch.equal(p, eng.select_smallest(ref_s, b)), (n, b)


@pytest.mark.parametrize("c", [1000, 260])
def test_badge_factors_sharded_on_one_gpu(eng, c):
    """badge_factors(row0=, n_total=) as the sharded loader calls it: uneven shards of a 10 037-row pool (short last
    batch of 53 at bs = 128), one boundary inside that batch, two shards long enough for the pipelined kernel.  The
    concatenated shards are bit-equal to the whole-pool call, which is equal on the pipelined and the direct route and
    within badge_factors64's bound."""
    n_total, bs = 10037, 128
    rng = np.random.default_rng(c)
    z = (rng.standard_normal((n_total, c)) * 3).astype(np.float32)
    dev = torch.from_numpy(z).cuda()
    whole_a, whole_n = eng.badge_factors(dev, bs)
    slab = torch.full((n_total, c + 4), float("nan"), device="cuda")
    slab[:, :c] = dev
    da, dn = eng.badge_factors(slab[:, :c], bs)
    assert torch.equal(bits(da), bits(whole_a)) and torch.equal(bits(dn), bits(whole_n))
    bounds = [0, 4100, 5000, 10000, n_total]
    parts = [eng.badge_factors(dev[lo:hi], bs, row0=lo, n_total=n_total) for lo, hi in zip(bounds[:-1], bounds[1:])]
    assert torch.equal(bits(torch.cat([p[0] for p in parts])), bits(whole_a))
    assert torch.equal(bits(torch.cat([p[1] for p in parts])), bits(whole_n))
    rows = np.unique(np.concatenate([rng.choice(n_total, 300, replace=False), np.arange(9950, n_total)]))
    a1, _ = R.badge_factors64(z[rows], 1)
    e1, en1 = R.badge_bound(z[rows], 1, "vec")
    bsz = R.batch_sizes(n_total, bs)[rows][:, None]
    check_within("K2 factors", whole_a.cpu().numpy()[rows, :c], a1 / bsz, e1 / bsz)
    check_within("K2 norm2", whole_n.cpu().numpy()[rows], (a1 ** 2).sum(1) / bsz[:, 0] ** 2, en1 / bsz[:, 0] ** 2)
    lo = 5000                                               # the shard form of the reference agrees with the whole
    ra, _ = R.badge_factors64(z[lo:10000], bs, row0=lo, n_total=n_total)
    wa, _ = R.badge_factors64(z, bs)
    np.testing.assert_array_equal(ra, wa[lo:10000])


@pytest.mark.parametrize("c", [1, 3, 7, 15, 16, 17, 100, 1000, 4000])
def test_pooled_embedding_against_fp64(eng, c):
    """K2p at class counts around the pooling height (16) and up to 4000, where the kernel's shared memory passes 48 KB;
    embedding widths around the pooling width; a short last loader batch (300 = 2 * 128 + 44)."""
    n, bs = 300, 128
    rng = np.random.default_rng(c)
    z = (rng.standard_normal((n, c)) * 3).astype(np.float32)
    ph = min(16, c)
    for d in (1, 31, 2048, 2049):
        h = np.maximum(rng.standard_normal((n, d)), 0).astype(np.float32)
        got = eng.badge_pooled_embedding(torch.from_numpy(z).cuda(), torch.from_numpy(h).cuda(), bs).cpu().numpy()
        w = ph * (512 // ph)
        assert got.shape == (n, (w + 3) & ~3) and (got[:, w:] == 0).all()
        check_within("K2p", got[:, :w], R.pooled64(z, h, bs), R.pooled_bound(z, h, bs))


def test_row_norms_scalar_and_vector_branches(eng):
    rng = np.random.default_rng(7)
    for d, kind in ((1, "scalar"), (3, "scalar"), (37, "scalar"), (4, "vec"), (36, "vec"), (128, "vec"), (2048, "vec")):
        x = (rng.standard_normal((1000, d)) * rng.choice([1e-3, 1.0, 1e3], (1000, 1))).astype(np.float32)
        got = eng.row_norm2(torch.from_numpy(x).cuda()).cpu().numpy()
        check_within("row_norm2 " + kind, got, R.row_norm2_64(x), R.row_norm2_bound(x, kind == "vec"))
    x = rng.standard_normal((1000, 64)).astype(np.float32)
    slab = torch.zeros((1000, 72), device="cuda")
    slab[:, 1:65] = torch.from_numpy(x).cuda()
    view = slab[:, 1:65]
    assert view.data_ptr() % 16 == 4
    check_within("row_norm2 scalar", eng.row_norm2(view).cpu().numpy(), R.row_norm2_64(x), R.row_norm2_bound(x, False))


@pytest.mark.parametrize("c", [1000, 37])
def test_host_buffer_tail_chunks(eng, c):
    """uncertainty_query_host streams the pool in chunks of 32 MiB / (4 c) rows: a last chunk below 4096 rows (the
    direct kernel after pipelined ones at c = 1000; the generic kernel throughout at c = 37) and tie groups across
    chunk boundaries, with the budget cutting through them: equal to the device path."""
    chunk = (32 << 20) // (4 * c)
    n = 2 * chunk + 1000 if c == 1000 else chunk + 1000
    rng = np.random.default_rng(c)
    z = (rng.standard_normal((n, c)) * 3).astype(np.float32)
    for edge in range(chunk, n - 1000 + 1, chunk):
        z[edge - 8:edge + 8] = z[edge - 8]                  # one tie group straddles every chunk boundary
    host = torch.from_numpy(z).pin_memory()
    dev = torch.from_numpy(z).cuda()
    for mode in (O.MODE_MARGIN, O.MODE_ENTROPY):
        s = eng.score_softmax(dev, mode)
        rank = eng.select_smallest(s, n).cpu().numpy()
        where = np.empty(n, dtype=np.int64)
        where[rank] = np.arange(n)
        budgets = {n, 1}
        for edge in range(chunk, n - 1000 + 1, chunk):
            budgets.add(int(where[edge - 8:edge + 8].min()) + 9)
        for b in sorted(budgets):
            assert np.array_equal(eng.uncertainty_query_host(host, mode, b), rank[:b]), (mode, b)
