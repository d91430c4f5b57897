"""CALSampler on the H100 (K18, K19 and the query around them) against the NumPy statement in cal_oracle.py: K18 bit for
bit, K19 within the bound of DESIGN section 4, the picks as K1b orders the device's scores."""
import numpy as np
import pytest
import torch

import cal_oracle as CO
from helpers import make_strategy
from test_cal import _EncoderNet

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from active_learning_b200.engine import Engine
    return Engine()


def _rows(n, m, d, seed):
    """Clustered rows of mixed norms; a candidate equal to a reference (d2 = 0), duplicated references, and references one
    fp32 ulp apart in one column (near-ties), placed before and after the row they copy."""
    rng = np.random.default_rng(seed)
    c = rng.normal(size=(12, d))
    x = (c[rng.integers(0, 12, n)] + 0.5 * rng.normal(size=(n, d))) * 10.0 ** rng.uniform(-2, 2, size=(n, 1))
    y = (c[rng.integers(0, 12, m)] + 0.5 * rng.normal(size=(m, d))) * 10.0 ** rng.uniform(-2, 2, size=(m, 1))
    x, y = x.astype(np.float32), y.astype(np.float32)
    if m >= 8:
        y[m - 1] = y[2]
        y[0] = y[m // 2]
        y[4] = y[3]
        y[4, 0] = np.nextafter(y[3, 0], np.float32(np.inf))
        y[5] = y[6]
        y[5, d - 1] = np.nextafter(y[6, d - 1], np.float32(-np.inf))
        for i in range(0, min(n, 40), 4):                       # candidates next to the near-ties
            x[i] = y[3 + (i // 4) % 4]
    x[n // 2] = y[m - 1]                                        # d2 = 0
    return x, y


@pytest.mark.parametrize("k", [1, 10, 32])
@pytest.mark.parametrize("d", [4, 28, 64, 520, 2048])
def test_knn_equals_the_oracle_bit_for_bit(eng, d, k):
    for m in sorted({1, max(1, k - 1), k, 127, 128, 129, 5000}):
        x, y = _rows(1037, m, d, d * 100 + k + m)
        want_i, want_d = CO.knn(x, y, k)
        yt = torch.from_numpy(y).cuda()
        for n in (1, 127, 128, 129, 1037):                      # rows are independent: a prefix of the same rows
            idx, d2, _ = eng.knn(torch.from_numpy(x[:n]).cuda(), yt, k)
            assert idx.cpu().numpy().tolist() == want_i[:n].tolist(), (m, n)
            assert (d2.cpu().numpy().view(np.uint64) == want_d[:n].view(np.uint64)).all(), (m, n)


def test_fallback_rows_are_exact(eng):
    """More than S = 32 identical references around the candidates' nearest, with an identical lower-indexed row before
    them and one after: the screen cannot certify those rows, the exact scan takes them."""
    rng = np.random.default_rng(4)
    d, m = 64, 3000
    y = rng.normal(size=(m, d)).astype(np.float32)
    v = rng.normal(size=d).astype(np.float32)
    y[7] = v
    y[100:160] = v
    y[2500] = v
    x = (v + 1e-3 * rng.normal(size=(300, d))).astype(np.float32)
    x[150:] = rng.normal(size=(150, d)).astype(np.float32)     # ordinary rows next to them
    for k in (1, 10, 32):
        idx, d2, fb = eng.knn(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), k)
        want_i, want_d = CO.knn(x, y, k)
        assert fb > 0 and fb <= 300
        assert idx.cpu().numpy().tolist() == want_i.tolist()
        assert (d2.cpu().numpy().view(np.uint64) == want_d.view(np.uint64)).all()
        assert idx[0, 0].item() == 7                            # the lower-indexed tie comes first


def _score_case(rng, n, m, c, k, scale):
    zc = (rng.normal(size=(n, c)) * scale).astype(np.float32)
    zr = (rng.normal(size=(m, c)) * scale).astype(np.float32)
    zc[:, 0] = np.clip(zc[:, 0] * 40, -80, 80)                 # logits of large magnitude
    zr[1:4] = zr[0]
    zc[0] = zr[0]
    idx = rng.integers(0, m, size=(n, k)).astype(np.int32)
    idx[0] = np.arange(k) % 4                                   # neighbours equal to the candidate: a zero score
    idx[1, k // 2:] = -1                                        # skipped entries
    idx[2, :] = -1
    return zc, zr, idx


@pytest.mark.parametrize("c", [2, 10, 1000])
@pytest.mark.parametrize("k", [1, 10, 32])
def test_scores_within_the_bound_and_keys_of_the_devices_scores(eng, c, k):
    rng = np.random.default_rng(c * 7 + k)
    zc, zr, idx = _score_case(rng, 3000, 700, c, k, 3.0)
    score, key = eng.cal_scores(torch.from_numpy(zc).cuda(), torch.from_numpy(zr).cuda(), torch.from_numpy(idx).cuda())
    score, key = score.cpu().numpy(), key.cpu().numpy()
    want = CO.scores(zc, zr, idx)
    bound = CO.score_bound(zc, zr, idx, want)
    assert np.isfinite(want).all() and (np.abs(score - want) <= bound).all()
    assert score[0] == 0.0 and score[2] == 0.0
    assert (key.view(np.uint32) == CO.keys(score).view(np.uint32)).all()
    assert not np.signbit(key[key == 0]).any()


def _query_case(eng, cache, seed=0):
    n, d, c = 6000, 36, 10
    rng = np.random.default_rng(seed)
    emb = torch.from_numpy(rng.integers(-4, 5, size=(n, d)).astype(np.float32))
    net = _EncoderNet(emb, c, seed)
    ev = rng.choice(n, 50, replace=False)
    lab = rng.choice(np.setdiff1d(np.arange(n), ev), 40, replace=False)
    s = make_strategy("CALSampler", torch.zeros(n, c), emb, ev, lab, 256, engine=eng, freeze_feature=cache,
                      cache_embeddings=cache)
    s.net = s.feature_net = net
    return s, net, emb


@pytest.mark.parametrize("cache", [True, False])
def test_query_over_two_rounds(eng, cache):
    s, net, emb = _query_case(eng, cache)
    for rnd, budget in enumerate((120, 700)):
        with torch.no_grad():
            logits = torch.nn.functional.linear(emb, net.linear.weight.cpu(), net.linear.bias.cpu())
        np.random.seed(100 + rnd)
        state = np.random.get_state()
        got, k = s.query(budget)
        after = np.random.get_state()
        np.random.set_state(state)
        union = np.asarray(s.get_idxs_for_coreset(), dtype=np.int64)
        assert (np.random.get_state()[1] == after[1]).all() and np.random.get_state()[2] == after[2]
        is_lab = s.already_labeled_idxs(boolean=True)[union]
        avail = s.available_query_idxs(boolean=True)[union]
        lab, cand = np.flatnonzero(is_lab), np.flatnonzero(avail)
        e, z = emb.numpy()[union], logits.numpy()[union]
        # the device's own scores, ordered by K1b's rule
        idx, _, _ = eng.knn(torch.from_numpy(e[cand]).cuda(), torch.from_numpy(e[lab]).cuda(), min(10, len(lab)))
        _, key = eng.cal_scores(torch.from_numpy(z[cand]).cuda(), torch.from_numpy(z[lab]).cuda(), idx)
        assert got == union[cand[CO.select(key.cpu().numpy(), budget)]].tolist() and k == budget
        # the oracle's picks, where its fp32 scores at the cut are more than 2 ulps apart
        want = CO.query_positions(e, z, is_lab, avail, budget)
        oi, _ = CO.knn(e[cand], e[lab], min(10, len(lab)))
        ok = CO.alq_ord(CO.keys(CO.scores(z[cand], z[lab], oi)))
        srt = np.sort(ok)
        assert int(srt[budget]) - int(srt[budget - 1]) > 2
        assert sorted(got) == sorted(union[want].tolist())
        rank = ok[np.searchsorted(union[cand], got)].astype(np.int64)
        assert (np.diff(rank) >= -2).all()
        s.update(got, k)
        s.round += 1
        with torch.no_grad():
            net.linear.bias.add_(1.0)


def test_imagenet_scale_on_sampled_rows(eng):
    n, m, d, k, c = 80000, 50000, 2048, 10, 1000
    g = torch.Generator(device="cuda").manual_seed(5)
    cen = torch.randn(300, d, device="cuda", generator=g)
    x = cen[torch.randint(0, 300, (n,), device="cuda", generator=g)] + 0.6 * torch.randn(n, d, device="cuda", generator=g)
    y = cen[torch.randint(0, 300, (m,), device="cuda", generator=g)] + 0.6 * torch.randn(m, d, device="cuda", generator=g)
    idx, d2, fb = eng.knn(x, y, k)
    zc = torch.randn(n, c, device="cuda", generator=g) * 3
    zr = torch.randn(m, c, device="cuda", generator=g) * 3
    score, _ = eng.cal_scores(zc, zr, idx)
    rows = np.sort(np.random.default_rng(6).choice(n, 2000, replace=False))
    xs, yh = x[torch.from_numpy(rows).cuda()].cpu().numpy(), y.cpu().numpy()
    want_i, want_d = CO.knn(xs, yh, k)
    assert idx.cpu().numpy()[rows].tolist() == want_i.tolist()
    assert (d2.cpu().numpy()[rows].view(np.uint64) == want_d.view(np.uint64)).all()
    zcs, zrh = zc[torch.from_numpy(rows).cuda()].cpu().numpy(), zr.cpu().numpy()
    want = CO.scores(zcs, zrh, want_i)
    assert (np.abs(score.cpu().numpy()[rows] - want) <= CO.score_bound(zcs, zrh, want_i, want)).all()


def test_errors_are_clean_and_leave_the_context_usable(eng):
    from active_learning_b200._lib import AlqError
    x = torch.randn(300, 16, device="cuda")
    y = torch.randn(200, 16, device="cuda")
    for k in (0, 33):
        with pytest.raises(AlqError, match=f"k={k}"):
            eng.knn(x, y, k)
    with pytest.raises(AlqError, match="d=6"):
        eng.knn(x[:, :6], y[:, :6], 3)
    with pytest.raises(AlqError, match="m=0"):
        eng.knn(x, y[:0], 3)
    for bad in (float("nan"), float("inf"), 1e20):
        yb = y.clone()
        yb[7, 3] = bad
        with pytest.raises(AlqError, match="1 rows have a squared norm"):
            eng.knn(x, yb, 3)
    with pytest.raises(AlqError, match="k=33"):
        eng.cal_scores(torch.randn(5, 4, device="cuda"), torch.randn(6, 4, device="cuda"),
                       torch.zeros(5, 33, dtype=torch.int32, device="cuda"))
    s, _, _ = _query_case(eng, False)
    s.idxs_lb[:] = False
    with pytest.raises(ValueError, match="CALSampler needs labeled rows"):
        s.query(10)
    idx, d2, _ = eng.knn(x, y, 5)
    want_i, want_d = CO.knn(x.cpu().numpy(), y.cpu().numpy(), 5)
    assert idx.cpu().numpy().tolist() == want_i.tolist()
    assert (d2.cpu().numpy().view(np.uint64) == want_d.view(np.uint64)).all()
