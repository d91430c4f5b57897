"""TypiClustSampler on the H100 (K15, K16, K17 and the k-means around them) against the NumPy statement in
typiclust_oracle.py, bit for bit."""
import numpy as np
import pytest
import torch

import typiclust_oracle as T
from helpers import make_strategy

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from active_learning_b200.engine import Engine
    return Engine()


def _clustered(n, d, k, seed, noise=0.3):
    rng = np.random.default_rng(seed)
    c = rng.normal(size=(k, d))
    return (c[rng.integers(0, k, n)] + noise * rng.normal(size=(n, d))).astype(np.float32)


def _exact_rows(rng, n, d, nnz=4):
    """Rows with `nnz` entries of +-1 (normalised: +-1/2 exactly), grouped around a few patterns so that clusters form;
    every fp32 norm and dot product of them is exact, so the D^2 seeding equals the oracle's on any hardware."""
    pats = [rng.choice(d, 8, replace=False) for _ in range(max(2, n // 200))]
    x = np.zeros((n, d), dtype=np.float32)
    for i in range(n):
        cols = rng.choice(pats[rng.integers(len(pats))], nnz, replace=False)
        x[i, cols] = rng.choice([-1.0, 1.0], nnz)
    return x


def _centres(rng, xhat, k):
    """Means of a few rows (norm < 1), then exact ties: duplicated centres, and copies one fp32 ulp away in one column,
    placed both before and after the centre they copy."""
    cen = np.stack([xhat[rng.choice(len(xhat), int(rng.integers(1, 6)), replace=False)].astype(np.float64).mean(0)
                    for _ in range(k)]).astype(np.float32)
    if k >= 8:
        cen[k - 1] = cen[0]
        cen[1] = cen[k - 2]
        cen[3] = cen[2]
        cen[3, 0] = np.nextafter(cen[2, 0], np.float32(2))
        cen[4] = cen[5]
        cen[4, 1] = np.nextafter(cen[5, 1], np.float32(-2))
    return cen


@pytest.mark.parametrize("d,k", [(d, k) for d in (4, 28, 64, 520, 2048) for k in (1, 127, 128, 129, 500, 700)]
                         + [(4, 32768), (64, 32768)])                  # K_MAX: 256 centre tiles
def test_assign_labels_equal_the_exact_argmin(eng, d, k):
    rng = np.random.default_rng(d * 1000 + k)
    n = 1037                                                            # a partial last row tile
    xhat = T.normalize(_clustered(n, d, 24, d + k))
    cen = _centres(rng, xhat, k)
    if k >= 8:
        cen[6] = xhat[10]                                               # a centre on a row: d2 = 0
    labels, changed, rech = eng.kmeans_assign(torch.from_numpy(xhat).cuda(), torch.from_numpy(cen).cuda())
    want = T.assign(xhat, cen)
    assert labels.cpu().numpy().tolist() == want.tolist()
    assert changed == n
    if k >= 8:
        assert rech > 0                                                 # the tied centres reach the recheck
    again, changed2, _ = eng.kmeans_assign(torch.from_numpy(xhat).cuda(), torch.from_numpy(cen).cuda(), labels)
    assert changed2 == 0 and again.cpu().numpy().tolist() == want.tolist()


def test_assign_rechecks_random_rows(eng):
    xhat = T.normalize(np.random.default_rng(5).normal(size=(20000, 2048)).astype(np.float32))
    cen = _centres(np.random.default_rng(6), xhat, 300)[8:]
    labels, _, rech = eng.kmeans_assign(torch.from_numpy(xhat).cuda(), torch.from_numpy(cen).cuda())
    assert rech > 0
    assert labels.cpu().numpy().tolist() == T.assign(xhat, cen).tolist()


@pytest.mark.parametrize("n,d,k", [(1, 4, 1), (1037, 28, 40), (5000, 2048, 700)])
def test_update_equals_the_sequential_means(eng, n, d, k):
    rng = np.random.default_rng(n + d)
    xhat = T.normalize(_clustered(n, d, 10, n))
    labels = rng.integers(0, max(1, k - k // 7), n)                     # the top clusters stay empty ...
    labels[rng.random(n) < 0.05] = 3 % k                                # ... and one is large
    cen = rng.normal(size=(k, d)).astype(np.float32)
    got = eng.kmeans_update(torch.from_numpy(xhat).cuda(), torch.from_numpy(labels.astype(np.int32)).cuda(),
                            torch.from_numpy(cen).cuda())
    assert (got.cpu().numpy().view(np.uint32) == T.update(xhat, labels, cen).view(np.uint32)).all()


def test_typicality_and_argmax_equal_the_oracle(eng):
    rng = np.random.default_rng(7)
    xhat = T.normalize(_clustered(12000, 64, 6, 7, noise=0.5))
    sizes = [1, 2, 3, 41, 5000, 64, 65]
    rows, goff = [], [0]
    for m in sizes:
        r = np.sort(rng.choice(len(xhat), m, replace=False))
        rows.append(r)
        goff.append(goff[-1] + m)
    xhat[rows[3][5]] = xhat[rows[3][9]]                                # duplicates: zero distances
    xhat[rows[4][:30]] = xhat[rows[4][100]]
    xhat[rows[2][1]] = xhat[rows[2][2]]
    flat = np.concatenate(rows)
    for kk in (20, 1, 32):
        typ, best = eng.typicality(torch.from_numpy(xhat).cuda(), torch.from_numpy(flat.astype(np.int32)).cuda(), goff, kk)
        typ = typ.cpu().numpy()
        for g, r in enumerate(rows):
            want = T.typicality(xhat, r, kk)
            assert typ[goff[g]:goff[g + 1]].tolist() == want.tolist(), (kk, g)
            assert best[g] == goff[g] + int(np.argmax(want))


def _seed_rows_of(eng):
    def seed_rows(xhat, first, unif, k):
        _, _, _, seeds = eng.kmeans(torch.from_numpy(xhat).cuda(), first, unif, k, max_iter=1)
        return seeds
    return seed_rows


@pytest.mark.parametrize("n,d,k", [(3000, 36, 50), (5000, 2048, 200)])
def test_seeding_equals_the_oracle_on_exact_rows(eng, n, d, k):
    rng = np.random.default_rng(n)
    xhat = T.normalize(_exact_rows(rng, n, d))
    first, unif = int(rng.integers(n)), rng.random(k - 1)
    assert _seed_rows_of(eng)(xhat, first, unif, k).tolist() == T.seed(xhat, first, unif, k).tolist()


@pytest.mark.parametrize("n,d,k", [(2000, 64, 20), (4000, 520, 500), (5000, 2048, 100)])
def test_kmeans_equals_the_oracle(eng, n, d, k):
    rng = np.random.default_rng(d)
    xhat = T.normalize(_clustered(n, d, max(2, k // 3), d))
    first, unif = int(rng.integers(n)), rng.random(k - 1)
    labels, centres, it, seeds = eng.kmeans(torch.from_numpy(xhat).cuda(), first, unif, k)
    want_l, want_c, want_it = T.lloyd(xhat, xhat[seeds].copy())
    assert seeds[0] == first and len(set(seeds.tolist())) == k
    assert it == want_it
    assert labels.cpu().numpy().tolist() == want_l.tolist()
    assert (centres.cpu().numpy().view(np.uint32) == want_c.view(np.uint32)).all()


def _e2e(eng, n, d, cache, seed=0):
    rng = np.random.default_rng(seed)
    emb = torch.from_numpy(_exact_rows(rng, n, d))
    ev = rng.choice(n, 50, replace=False)
    lab = rng.choice(np.setdiff1d(np.arange(n), ev), 40, replace=False)
    s = make_strategy("TypiClustSampler", torch.zeros(n, 4), emb, ev, lab, 256, engine=eng, freeze_feature=cache,
                      cache_embeddings=cache)
    return s, emb


@pytest.mark.parametrize("cache", [True, False])
def test_query_equals_the_oracle_over_two_rounds(eng, cache):
    s, emb = _e2e(eng, 6000, 36, cache)
    for rnd, budget in enumerate((120, 700)):
        np.random.seed(100 + rnd)
        state = np.random.get_state()
        got, k = s.query(budget)
        after = np.random.get_state()
        np.random.set_state(state)
        union = np.asarray(s.get_idxs_for_coreset(), dtype=np.int64)
        is_lab = s.already_labeled_idxs(boolean=True)[union]
        avail = s.available_query_idxs(boolean=True)[union]
        want = union[T.query_positions(emb.numpy()[union], is_lab, avail, budget)].tolist()
        assert got == want and k == budget
        assert (np.random.get_state()[1] == after[1]).all() and np.random.get_state()[2] == after[2]
        s.update(got, k)
        s.round += 1


def test_imagenet_scale_fixed_point_and_typicalities(eng):
    n, d, k = 130000, 2048, 500
    rng = np.random.default_rng(11)
    x = _clustered(n, d, 300, 11, noise=0.6)
    xt = torch.from_numpy(x).cuda()
    xhat_t = eng.normalize(xt)
    xhat = xhat_t.cpu().numpy()
    sample = rng.choice(n, 4000, replace=False)
    assert (xhat[sample].view(np.uint32) == T.normalize(x[sample]).view(np.uint32)).all()
    labels_t, centres_t, it, seeds = eng.kmeans(xhat_t, int(rng.integers(n)), rng.random(k - 1), k)
    labels, centres = labels_t.cpu().numpy().astype(np.int64), centres_t.cpu().numpy()
    assert it <= T.MAX_ITER
    if it < T.MAX_ITER:                                                 # converged: a fixed point
        assert (T.assign(xhat[sample], centres) == labels[sample]).all()
        for c in rng.choice(np.unique(labels), 12, replace=False):
            rows = np.flatnonzero(labels == c)
            s = np.cumsum(xhat[rows].astype(np.float64), axis=0)[-1]
            assert (centres[c] == (s / len(rows)).astype(np.float32)).all()
    # one cycle of the walk over every cluster, as the sampler launches it
    order = T.cluster_order(labels, np.zeros(n, dtype=bool), k)
    rows = [np.flatnonzero(labels == c) for c in order]
    goff = np.concatenate([[0], np.cumsum([len(r) for r in rows])])
    flat = np.concatenate(rows)
    typ, best = eng.typicality(xhat_t, torch.from_numpy(flat.astype(np.int32)).cuda(), goff, T.K_NN)
    typ = typ.cpu().numpy()
    for g in rng.choice(len(order), 8, replace=False):
        want = T.typicality(xhat, rows[g])
        assert typ[goff[g]:goff[g + 1]].tolist() == want.tolist()
        assert best[g] == goff[g] + int(np.argmax(want))


def test_errors_are_clean_and_leave_the_context_usable(eng):
    from active_learning_b200._lib import AlqError
    x = torch.randn(300, 16, device="cuda")
    y = x.clone()
    y[7, 3] = float("nan")
    with pytest.raises(ValueError):
        eng.normalize(y)
    y[7, 3] = float("inf")
    with pytest.raises(ValueError):
        eng.normalize(y)
    xhat = eng.normalize(x)
    rows = torch.arange(300, dtype=torch.int32, device="cuda")
    with pytest.raises(AlqError, match="k=33"):
        eng.typicality(xhat, rows, [0, 300], 33)
    with pytest.raises(AlqError):
        eng.typicality(xhat, rows, [0, 0, 300], 20)                      # an empty group
    with pytest.raises(ValueError):
        eng.kmeans(xhat, 0, np.zeros(300), 301)
    shifted = torch.empty(300 * 16 + 1, device="cuda")[1:].view(300, 16)   # contiguous, 4 bytes off 16-byte alignment
    shifted.copy_(xhat)
    with pytest.raises(AlqError, match="xhat / hi / lo not 16-byte aligned"):
        eng.kmeans_assign(shifted, xhat[:20].clone())                    # K15's recheck reads xhat as float4
    typ, best = eng.typicality(xhat, rows, [0, 300], 32)
    want = T.typicality(xhat.cpu().numpy(), np.arange(300), 32)
    assert typ.cpu().numpy().tolist() == want.tolist() and best[0] == int(np.argmax(want))
