"""K15, K16 and K21 at the cluster counts their limits admit, against typiclust_oracle.py and alfamix_oracle.py bit for
bit.  K16 keeps 4 bytes per cluster of dynamic shared memory per chunk: up to K = 12 288 that fits the default 48 KB,
from K = 12 289 the kernels run on the opt-in, and K_MAX = 32 768 needs 128 KB.  K = 32 769 is refused."""
import numpy as np
import pytest
import torch

import alfamix_oracle as AO
import probcover_oracle as P
import typiclust_oracle as T
from test_gpu_typiclust import _clustered

pytestmark = pytest.mark.gpu

K_MAX = 32768
OUTSIDE = (-1, -7, 2 ** 31 - 1)                                         # labels that name no cluster (and K, K + 1)


@pytest.fixture(scope="module")
def eng():
    from active_learning_b200.engine import Engine
    return Engine()


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("k", [12288, 12289, K_MAX])                    # 4 K = 49 152, 49 156 and 131 072 bytes
@pytest.mark.parametrize("n,d", [(5 * 1024 + 37, 8), (40 * 1024 + 517, 36)])
def test_update_across_the_shared_memory_opt_in(eng, n, d, k):
    rng = np.random.default_rng(n + k)
    xhat = T.normalize(_clustered(n, d, 10, n))
    labels = rng.integers(0, k, n)
    labels[(labels >= k - 200) & (labels < k - 1)] = 0                  # empty clusters just below the last one ...
    labels[rng.random(n) < 0.1] = k - 1                                 # ... which is large
    single = rng.choice(np.arange(1, k - 200), 40, replace=False)
    labels[np.isin(labels, single)] = 0
    rows = rng.choice(n, 40 + 5 * len(OUTSIDE), replace=False)
    labels[rows[:40]] = single                                          # clusters of one row
    labels[rows[40:]] = np.resize(OUTSIDE + (k, k + 1), 5 * len(OUTSIDE))   # rows K16 skips
    size = np.bincount(labels[(labels >= 0) & (labels < k)], minlength=k)
    assert (size[single] == 1).all() and (size[k - 200:k - 1] == 0).all() and size[k - 1] > n // 20
    cen = rng.normal(size=(k, d)).astype(np.float32)
    got = eng.kmeans_update(_cuda(xhat), _cuda(labels.astype(np.int32)), _cuda(cen))
    assert (got.cpu().numpy().view(np.uint32) == T.update(xhat, labels, cen).view(np.uint32)).all()


def test_kmeans_nearest_at_k_max(eng):
    n, d, k = 40000, 36, K_MAX
    rng = np.random.default_rng(21)
    xhat = T.normalize(_clustered(n, d, 400, 21))
    labels = rng.integers(0, k, n)
    labels[(labels >= 1000) & (labels < 1100)] = k - 1                  # empty clusters
    centres = T.normalize(_clustered(k, d, 400, 22))
    on = rng.choice(n, 3000, replace=False)
    centres[labels[on]] = xhat[on]                                      # centres on one of their rows: d2 = 0
    rest = rng.permutation(np.setdiff1d(np.arange(n), on))
    dup, out = rest[:1500], rest[1500:1500 + 50]
    xhat[dup] = xhat[on[:1500]]                                         # duplicates in the same cluster, before and
    labels[dup] = labels[on[:1500]]                                     # after their copy: ties go to the lowest row
    labels[out] = np.resize(OUTSIDE + (k, k + 1), len(out))
    got = eng.kmeans_nearest(_cuda(xhat), _cuda(labels.astype(np.int32)), _cuda(centres))
    keep = np.flatnonzero((labels >= 0) & (labels < k))                 # the oracle indexes centres[labels]
    want = AO.nearest(xhat[keep], labels[keep], centres)
    want = np.where(want >= 0, keep[np.maximum(want, 0)], -1)
    zero = P.exact_d2(xhat[keep], centres[labels[keep]]) == 0
    assert np.bincount(labels[keep][zero], minlength=k).max() >= 2      # tied rows at d2 = 0 exist
    assert got.tolist() == want.tolist() and (got[1000:1100] == -1).all() and got[k - 1] >= 0


def test_k_past_the_cap_is_refused_and_leaves_the_context_usable(eng):
    from active_learning_b200._lib import AlqError
    n, d = 3000, 8
    xhat = T.normalize(_clustered(n, d, 10, 4))
    x = _cuda(xhat)
    big = _cuda(T.normalize(_clustered(K_MAX + 1, d, 10, 5)))
    with pytest.raises(AlqError, match=r"alq_kmeans_assign: K=32769 outside \[1, 32768\]"):
        eng.kmeans_assign(x, big)
    before = big.clone()
    with pytest.raises(AlqError, match=r"alq_kmeans_update: K=32769 outside \[1, 32768\]"):
        eng.kmeans_update(x, torch.zeros(n, dtype=torch.int32, device="cuda"), big)
    assert torch.equal(big, before)
    cen = xhat[::60].copy()
    labels, _, _ = eng.kmeans_assign(x, _cuda(cen))
    want = T.assign(xhat, cen)
    assert labels.cpu().numpy().tolist() == want.tolist()
    got = eng.kmeans_update(x, labels, _cuda(cen))
    assert (got.cpu().numpy().view(np.uint32) == T.update(xhat, want, cen).view(np.uint32)).all()


def test_lloyd_through_the_opt_in(eng):
    n, d, k = 24000, 36, 16000                                           # 4 K = 64 000 bytes
    rng = np.random.default_rng(16)
    xhat = T.normalize(_clustered(n, d, 400, 16))
    first, unif = int(rng.integers(n)), rng.random(k - 1)
    labels, centres, it, seeds = eng.kmeans(_cuda(xhat), first, unif, k)
    want_l, want_c, want_it = T.lloyd(xhat, xhat[seeds].copy())
    assert len(set(seeds.tolist())) == k and it == want_it
    assert labels.cpu().numpy().tolist() == want_l.tolist()
    assert (centres.cpu().numpy().view(np.uint32) == want_c.view(np.uint32)).all()
