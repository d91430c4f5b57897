"""The claims behind the score-bucket route of the fused uncertainty tail (alq_score.cu, select_epilogue), restated in
NumPy fp32 and checked on the CPU.

The kernel orders the b winners without a global sort: with T the 22-bit key prefix of the b-th smallest score and
[lo, hi] = [lower edge of the first populated 11-bit key bin, upper edge of prefix T], a candidate goes to bucket
    q = clamp(floor((score - lo) * (G / (hi - lo))), 0, G - 1)            (fp32 arithmetic, G = CTAs)
and bucket q is sorted by CTA q alone; its winners take the ranks that follow the sizes of the buckets below.  That is
exact iff (1) the key <-> float maps are inverse order isomorphisms, (2) every candidate score lies in [lo, hi] and
(3) q is monotone (non-decreasing) in the key.  Ties / non-finite edges make the kernel leave the route; the
conditions under which it does so are restated here too."""
import numpy as np

G = 132                                 # one CTA per SM of an H100


def ord_key(f32):                       # alq_ord (alq_common.cuh): monotone float -> uint32
    u = f32.view(np.uint32)
    return np.where(u & 0x80000000, ~u, u | 0x80000000).astype(np.uint32)


def key_to_float(key):                  # sel_key_to_float
    key = key.astype(np.uint32)
    u = np.where(key & 0x80000000, key & 0x7FFFFFFF, ~key).astype(np.uint32)
    return u.view(np.float32)


def edges(keys, b):
    """lo / hi exactly as the epilogue derives them: first populated level-0 bin, prefix T of the b-th smallest key."""
    first_bin = int(keys.min() >> 21)
    t = int(np.sort(keys)[b - 1] >> 10)
    lo = key_to_float(np.array([first_bin << 21], dtype=np.uint32))[0]
    hi = key_to_float(np.array([(t << 10) | 0x3FF], dtype=np.uint32))[0]
    return lo, hi, t


def bucket(score, lo, hi):
    with np.errstate(all="ignore"):
        scale = np.float32(G) / np.float32(hi - lo)
        q = np.floor((score.astype(np.float32) - np.float32(lo)) * scale)
        return np.clip(np.nan_to_num(q, nan=0.0), 0, G - 1).astype(np.int64), scale


def test_key_maps_are_inverse_order_isomorphisms():
    rng = np.random.default_rng(0)
    with np.errstate(over="ignore"):
        f = np.concatenate([(rng.standard_normal(20000) * 10.0 ** rng.integers(-30, 30, 20000)).astype(np.float32),
                            np.array([0.0, 1e-45, -1e-45, np.inf, -np.inf, 3.4e38, -3.4e38, 1.0, -1.0], dtype=np.float32)])
    f = f + np.float32(0.0)                                   # the kernel keys `score + 0.0f`: -0.0 never appears
    k = ord_key(f)
    assert np.array_equal(key_to_float(k).view(np.uint32), f.view(np.uint32))
    order = np.argsort(f, kind="stable")
    assert np.all(np.diff(k[order].astype(np.int64)) >= 0)
    assert np.all((np.diff(f[order]) > 0) == (np.diff(k[order].astype(np.int64)) > 0))


def _pools(rng):
    n = 50000
    yield rng.random(n).astype(np.float32)                                        # margins of a flat model
    yield (rng.random(n) ** 6).astype(np.float32)                                 # piled up next to 0
    yield (1.0 - rng.random(n) ** 4).astype(np.float32)                           # piled up next to 1
    yield (-np.log(1000.0) * rng.random(n)).astype(np.float32)                    # negative entropies
    yield np.exp(rng.normal(-8, 5, n)).astype(np.float32)                         # 20 decades
    yield (rng.integers(0, 50, n) / np.float32(64)).astype(np.float32)            # heavy ties on a dyadic grid
    yield np.concatenate([np.full(n // 2, 0.25, np.float32), rng.random(n // 2).astype(np.float32)])


def test_bucket_is_monotone_and_ranks_follow_bucket_sizes():
    rng = np.random.default_rng(1)
    for pool in _pools(rng):
        scores = pool + np.float32(0.0)
        keys = ord_key(scores)
        for b in (1, 17, 5000, len(scores) // 2, len(scores)):
            lo, hi, t = edges(keys, b)
            cand = (keys >> 10) <= t
            cs, ck = scores[cand], keys[cand]
            assert cand.sum() >= b
            assert np.all(cs >= lo) and np.all(cs <= hi)                           # (2)
            q, scale = bucket(cs, lo, hi)
            spread = np.isfinite(lo) and np.isfinite(hi) and hi > lo and np.isfinite(scale)
            if not spread:
                continue                                                           # the kernel leaves the route
            order = np.argsort(ck, kind="stable")
            assert np.all(np.diff(q[order]) >= 0)                                  # (3) monotone in the key
            # ranks: sorting inside each bucket and concatenating the buckets IS the global order
            words = (ck.astype(np.uint64) << np.uint64(32)) | np.flatnonzero(cand).astype(np.uint64)
            by_bucket = np.concatenate([np.sort(words[q == g]) for g in range(G)])
            assert np.array_equal(by_bucket, np.sort(words))


def test_degenerate_pools_leave_the_route():
    """All-equal scores: hi - lo spans one 22-bit prefix (or a denormal next to 0): the scale overflows or the edges
    coincide, so `spread` is false -- or everything lands in one bucket, which the kernel detects from the counters."""
    for value in (0.0, 0.5, 1e-30, 123456.0):
        scores = np.full(4096, value, np.float32)
        keys = ord_key(scores)
        lo, hi, _ = edges(keys, 1000)
        q, scale = bucket(scores, lo, hi)
        spread = np.isfinite(lo) and np.isfinite(hi) and hi > lo and np.isfinite(scale)
        assert (not spread) or len(np.unique(q)) == 1
    nan = np.array([np.nan, 1.0, 2.0], dtype=np.float32)
    lo, hi, _ = edges(ord_key(nan), 3)                        # a NaN among the winners: the upper edge is not finite
    assert not np.isfinite(hi)
