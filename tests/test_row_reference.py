"""tests/row_reference.py (the float64 restatement of the streaming row kernels) against the torch oracle, scipy and the
reference's MASE goldens.  CPU only."""
import os

import numpy as np
import pytest
import torch
from scipy.special import entr

import row_reference as R
from oracle import al_oracle as O
from test_oracle_golden_mase import head_of, pool_of

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = (O.MODE_MARGIN, O.MODE_LEAST_CONFIDENCE, O.MODE_ENTROPY)


def special_rows(c, rng):
    """Rows where softmax kernels go wrong: masked classes, one finite logit, all -inf, NaN, +inf, +-3e38, gaps below
    -87 (exp flushes to zero in fp32), exact ties at the maximum, a large temperature."""
    rows = []
    r = rng.standard_normal(c) * 3
    r[1::3] = -np.inf
    rows.append(r)
    r = np.full(c, -np.inf)
    r[c // 2] = 1.5
    rows.append(r)
    rows.append(np.full(c, -np.inf))
    r = rng.standard_normal(c)
    r[min(1, c - 1)] = np.nan
    rows.append(r)
    r = rng.standard_normal(c)
    r[c - 1] = np.inf
    rows.append(r)
    rows.append(np.where(np.arange(c) % 2 == 0, 3e38, -3e38))
    r = np.full(c, -3e38)
    r[c // 3] = 3e38
    rows.append(r)
    r = -87.5 - 10 * rng.random(c)
    r[0] = 0.0
    r[c // 2:c // 2 + 2] = -80.0
    rows.append(r)
    rows.append(np.zeros(c))
    r = rng.standard_normal(c)
    r[0] = r[c - 1] = 5.0
    rows.append(r)
    rows.append(rng.standard_normal(c) * 50)
    r = rng.standard_normal(c)
    r[0], r[min(2, c - 1)] = np.inf, np.nan
    rows.append(r)
    return np.asarray(rows, dtype=np.float32)


def test_depths():
    assert R.sum_depth(4, "vec") == 9 and R.sum_depth(128, "vec") == 9 and R.sum_depth(129, "vec") == 13
    assert R.sum_depth(2048, "vec") == 69 and R.sum_depth(37, "generic") == 7 and R.sum_depth(4096, "generic") == 133


@pytest.mark.parametrize("c", [4, 10, 37, 132, 1000, 2048])
def test_softmax_scores64_against_the_torch_oracle(c):
    """The torch oracle (fp32, accurate exp) lies inside the kernel's bound around the fp64 scores, NaN exactly where
    the oracle is NaN; the bound is tighter than a blanket 2e-6 on ordinary rows."""
    rng = np.random.default_rng(c)
    z = np.concatenate([special_rows(c, rng), (rng.standard_normal((300, c)) * 3).astype(np.float32)])
    for mode in MODES:
        ref = R.softmax_scores64(z, mode)
        got = O.softmax_scores(torch.from_numpy(z), mode).double().numpy()
        assert np.array_equal(np.isnan(ref), np.isnan(got)), mode
        bound = R.score_bound(z, mode, "vec")
        assert np.array_equal(np.isnan(ref), np.isnan(bound))
        ok = ~np.isnan(ref)
        assert (np.abs(got - ref)[ok] <= bound[ok]).all(), (mode, np.max(np.abs(got - ref)[ok] / bound[ok]))
        if mode != O.MODE_ENTROPY:
            assert np.median(bound[12:]) < 2e-6, mode


def test_masked_and_extreme_rows_have_the_closed_form_scores():
    c = 8
    z = special_rows(c, np.random.default_rng(0))
    for mode in MODES:
        s = R.softmax_scores64(z, mode)
        assert np.isnan(s[[2, 3, 4, 11]]).all() and not np.isnan(np.delete(s, [2, 3, 4, 11])).any(), mode
    ent = R.softmax_scores64(z, O.MODE_ENTROPY)
    assert ent[1] == 0.0 and np.isclose(ent[5], -np.log(4)) and np.isclose(ent[8], -np.log(c))
    mar = R.softmax_scores64(z, O.MODE_MARGIN)
    assert mar[1] == 1.0 and mar[5] == 0.0 and mar[8] == 0.0 and mar[9] == 0.0 and mar[6] == 1.0


def test_entropy_matches_scipy_entr():
    rng = np.random.default_rng(1)
    c = 57
    z = np.concatenate([special_rows(c, rng), rng.standard_normal((200, c)) * 4])
    ent = R.softmax_scores64(z, O.MODE_ENTROPY)
    ok = ~np.isnan(ent)
    zz = z[ok].astype(np.float64)
    p = np.exp(zz - zz.max(1, keepdims=True))
    p /= p.sum(1, keepdims=True)
    np.testing.assert_allclose(ent[ok], -entr(p).sum(1), rtol=1e-12, atol=1e-300)


def test_masking_a_class_in_the_oracle_matches_the_reference():
    """O.softmax_scores(entropy) adopts 0 log 0 = 0: a -inf logit leaves the row finite and equal to the row without
    that class."""
    rng = np.random.default_rng(2)
    z = (rng.standard_normal((50, 20)) * 3).astype(np.float32)
    zm = z.copy()
    zm[::2, 7] = -np.inf
    got = O.softmax_scores(torch.from_numpy(zm), O.MODE_ENTROPY).numpy()
    assert np.isfinite(got).all()
    drop = O.softmax_scores(torch.from_numpy(np.delete(z, 7, axis=1)), O.MODE_ENTROPY).numpy()
    np.testing.assert_allclose(got[::2], drop[::2], rtol=1e-6)
    ref = R.softmax_scores64(zm, O.MODE_ENTROPY)
    assert (np.abs(got - ref) <= R.score_bound(zm, O.MODE_ENTROPY, "vec")).all()


def test_badge_factors64_against_the_oracle():
    rng = np.random.default_rng(3)
    z = (rng.standard_normal((300, 37)) * 3).astype(np.float32)
    a, an = R.badge_factors64(z, 128)
    ref = O.badge_factors(torch.from_numpy(z), 128).double().numpy()
    eg, en = R.badge_bound(z, 128, "generic")
    assert (np.abs(ref - a) <= eg).all()
    assert (np.abs((ref ** 2).sum(1) - an) <= en).all()
    # a shard of a longer loader pass: the rows of the short last batch take 1 / tail
    a2, _ = R.badge_factors64(z[100:], 128, row0=100, n_total=300)
    np.testing.assert_array_equal(a2, a[100:])


def test_pooled64_against_the_oracle():
    rng = np.random.default_rng(4)
    for c, d in ((10, 33), (37, 100), (3, 7)):
        z = (rng.standard_normal((70, c)) * 3).astype(np.float32)
        h = rng.standard_normal((70, d)).astype(np.float32)
        got = R.pooled64(z, h, 16)
        ref = O.gradient_embeddings(torch.from_numpy(z), torch.from_numpy(h), 16, use_adaptive_pool=True).double().numpy()
        assert got.shape == ref.shape
        assert (np.abs(got - ref) <= R.pooled_bound(z, h, 16) + 1e-12).all(), (c, d)


def test_row_norm_bound_holds_for_fp32_sums():
    rng = np.random.default_rng(5)
    x = rng.standard_normal((100, 37)).astype(np.float32)
    got = (x * x).sum(1, dtype=np.float32).astype(np.float64)
    assert (np.abs(got - R.row_norm2_64(x)) <= R.row_norm2_bound(x, False)).all()


def test_mase64_follows_torch_max_on_nan_rows():
    w = np.random.default_rng(6).standard_normal((5, 8))
    z = np.array([[1.0, np.nan, 3.0, np.nan, 0.0],
                  [np.inf, 0.0, np.nan, 1.0, 2.0],
                  [-np.inf] * 5,
                  [0.0, 2.0, 2.0, -np.inf, 1.0]], dtype=np.float32)
    mm, pred, r = R.mase64(z, w)
    assert pred.tolist() == torch.from_numpy(z).max(dim=1).indices.tolist() == [1, 2, 0, 1]
    assert np.isinf(r[:3]).all() and np.isinf(mm[:3]).all()
    assert mm[3] == 0.0 and np.isinf(r[3, 3]) and np.isinf(r[3, 1])
    rmm, rpc, rpred = O.mase_margins_closed_form(torch.from_numpy(z), torch.from_numpy(w).float())
    assert rpred.tolist() == pred.tolist() and torch.isinf(rmm[:3]).all()


@pytest.mark.parametrize("tag", ["a", "b", "t", "d"])
def test_mase64_reproduces_the_reference_golden(tag):
    g = dict(np.load(os.path.join(ROOT, "tests", "golden", "reference_golden_mase.npz")))
    pool = pool_of(g, tag)
    emb, w, b = head_of(g, tag)
    logits = torch.nn.functional.linear(emb[pool], w, b).numpy()
    mm, pred, r = R.mase64(logits, w.numpy())
    ref_pc, ref_mm = g[f"{tag}_per_class"], g[f"{tag}_min_margins"]
    assert np.array_equal(pred, g[f"{tag}_pred"])
    assert np.array_equal(np.isinf(r), np.isinf(ref_pc))
    fin = np.isfinite(ref_pc)
    np.testing.assert_allclose(r[fin], ref_pc[fin], rtol=1e-4, atol=2e-6)
    np.testing.assert_allclose(mm, ref_mm, rtol=1e-4, atol=2e-6)
    if tag == "d":
        assert int(np.isinf(r).sum(1).max()) == 2
