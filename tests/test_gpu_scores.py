"""K1 / K1b / K2 / K2p / row norms on the GPU, through the C ABI, against the oracle and the
golden vectors produced by the reference."""
import numpy as np
import pytest
import torch

from helpers import FUSED_TAIL_SHAPES, fused_tail_logits, skewed_tail_pools, tied_tail_pools
from oracle import al_oracle as O

pytestmark = pytest.mark.gpu

TOL_PROB = 2e-6      # north star: per-sample scores within 1e-4 fp32; we hold 2e-6


@pytest.fixture(scope="module")
def eng():
    from active_learning_b200.engine import Engine
    return Engine()


@pytest.mark.parametrize("n,c", [(1, 10), (257, 10), (300, 37), (1000, 1000), (513, 1024), (129, 2048),
                                 (64, 4096)])
def test_softmax_scores_match_oracle(eng, n, c):
    torch.manual_seed(n * 7 + c)
    logits = torch.randn(n, c) * 3.0
    dev = logits.cuda()
    for mode in (O.MODE_MARGIN, O.MODE_LEAST_CONFIDENCE, O.MODE_ENTROPY):
        got = eng.score_softmax(dev, mode).cpu()
        ref = O.softmax_scores(logits, mode)
        tol = TOL_PROB if mode != O.MODE_ENTROPY else 2e-5   # entropy is O(log C), same relative bar
        assert torch.allclose(got, ref, rtol=0, atol=tol), (mode, (got - ref).abs().max())


def test_scores_on_strided_slab(eng):
    """Row pitch != C (a view into a wider slab)."""
    torch.manual_seed(3)
    slab = torch.randn(500, 1024, device="cuda") * 3
    view = slab[:, :1000]
    got = eng.score_softmax(view, O.MODE_MARGIN).cpu()
    assert torch.allclose(got, O.softmax_scores(view.cpu(), O.MODE_MARGIN), rtol=0, atol=TOL_PROB)


def test_margin_ties_are_exact_zero(eng):
    rng = np.random.default_rng(0)
    logits = torch.from_numpy(rng.integers(-8, 9, size=(4000, 10)).astype(np.float32) / 4)
    got = eng.score_softmax(logits.cuda(), O.MODE_MARGIN).cpu()
    top2 = logits.topk(2, dim=1).values
    tied = top2[:, 0] == top2[:, 1]
    assert tied.sum() > 100 and (got[tied] == 0).all() and (got[~tied] > 0).all()


@pytest.mark.parametrize("n,b", [(1, 1), (100, 100), (4097, 1), (4097, 1365), (100000, 10000),
                                 (100000, 16384), (100000, 40000), (300000, 300000)])
def test_select_smallest_is_stable_sort_prefix(eng, n, b):
    rng = np.random.default_rng(n + b)
    # quantised scores: thousands of exact ties, including across the budget boundary
    scores = torch.from_numpy((rng.integers(0, max(2, n // 50), size=n) / 64.0).astype(np.float32))
    if n > 10:
        scores[rng.integers(0, n, 5)] = 0.0
        scores[rng.integers(0, n, 3)] = -0.0
        scores[rng.integers(0, n, 3)] = -1.5
    got = eng.select_smallest(scores.cuda(), b).cpu().numpy()
    assert np.array_equal(got, O.select_smallest(scores, b))


@pytest.mark.parametrize("n,b", [(1, 1), (37, 37), (4097, 1365), (80000, 10000), (100000, 16384), (262144, 5000)])
def test_select_cluster_and_multikernel_paths_agree(eng, n, b):
    """Both K1b implementations (one cluster-resident launch / multi-kernel radix select) against the oracle,
    on tie-heavy scores."""
    rng = np.random.default_rng(n * 3 + b)
    scores = torch.from_numpy((rng.integers(0, max(2, n // 40), size=n) / 32.0 - 1.0).astype(np.float32))
    ref = O.select_smallest(scores, b)
    try:
        for impl in (1, 2):
            eng.set_option("select_impl", impl)
            assert np.array_equal(eng.select_smallest(scores.cuda(), b).cpu().numpy(), ref), impl
    finally:
        eng.set_option("select_impl", 0)


def test_select_all_equal_scores(eng):
    scores = torch.full((50000,), 0.25)
    got = eng.select_smallest(scores.cuda(), 777).cpu().numpy()
    assert np.array_equal(got, np.arange(777))


def test_margin_and_confidence_match_reference_golden(eng, gold):
    n = int(gold["e2e_n"])
    lb = np.zeros(n, dtype=bool)
    lb[gold["e2e_labeled"]] = True
    for tag in ("f32_c10", "f32_c1000"):
        pool = O.available_query_idxs(lb, gold["e2e_eval_idxs"], shuffle=False)
        logits = torch.from_numpy(gold[f"margin_{tag}_logits"])[pool].cuda()
        pos = eng.select_smallest(eng.score_softmax(logits, O.MODE_MARGIN), 60).cpu().numpy()
        assert pool[pos].tolist() == gold[f"margin_{tag}_picks"].tolist()
    np.random.seed(7)
    pool = O.available_query_idxs(lb, gold["e2e_eval_idxs"], shuffle=True)
    logits = torch.from_numpy(gold["confidence_f32_logits"])[pool].cuda()
    pos = eng.select_smallest(eng.score_softmax(logits, O.MODE_LEAST_CONFIDENCE), 60).cpu().numpy()
    assert pool[pos].tolist() == gold["confidence_f32_picks"].tolist()


def test_host_buffer_entry_point_equals_device_path(eng):
    torch.manual_seed(5)
    logits = (torch.randn(30000, 1000) * 3).pin_memory()
    for mode in (O.MODE_MARGIN, O.MODE_ENTROPY):
        host = eng.uncertainty_query_host(logits, mode, 5000)
        dev = eng.select_smallest(eng.score_softmax(logits.cuda(), mode), 5000).cpu().numpy()
        assert np.array_equal(host, dev)
    pageable = torch.randn(3000, 10)
    assert np.array_equal(eng.uncertainty_query_host(pageable, O.MODE_LEAST_CONFIDENCE, 300),
                          O.select_smallest(O.softmax_scores(pageable, O.MODE_LEAST_CONFIDENCE), 300))


def test_badge_factors_match_oracle_and_reference(eng, gold):
    lg, hg = torch.from_numpy(gold["ge_logits"]), torch.from_numpy(gold["ge_emb"])
    a, an = eng.badge_factors(lg.cuda(), 16)
    a = a.cpu()
    assert a.shape == (53, 12) and (a[:, 10:] == 0).all()        # zero padding up to x4
    ref = O.badge_factors(lg, 16)
    assert torch.allclose(a[:, :10], ref, rtol=0, atol=1e-7)
    assert torch.allclose(an.cpu(), ref.square().sum(1), rtol=1e-5, atol=1e-9)
    full = (a[:, :10, None] * hg[:, None, :]).reshape(53, -1)    # the reference's materialised form
    np.testing.assert_allclose(full.numpy(), gold["ge_full"], rtol=0, atol=2e-7)
    torch.manual_seed(1)
    big = torch.randn(700, 1000) * 3                              # vector path, short last batch
    a, an = eng.badge_factors(big.cuda(), 128)
    ref = O.badge_factors(big, 128)
    assert torch.allclose(a.cpu(), ref, rtol=0, atol=1e-7)
    assert torch.allclose(an.cpu(), ref.square().sum(1), rtol=2e-5, atol=1e-10)


def test_pooled_embedding_matches_reference(eng, gold):
    for lk, ek, gk, bs in (("ge_logits", "ge_emb", "ge_pooled", 16), ("ge2_logits", "ge2_emb", "ge2_pooled", 4)):
        got = eng.badge_pooled_embedding(torch.from_numpy(gold[lk]).cuda(), torch.from_numpy(gold[ek]).cuda(), bs)
        w = gold[gk].shape[1]
        assert (got[:, w:] == 0).all()
        np.testing.assert_allclose(got.cpu().numpy()[:, :w], gold[gk], rtol=0, atol=3e-7)
    torch.manual_seed(2)
    lg, em = torch.randn(300, 1000) * 3, torch.relu(torch.randn(300, 2048))
    got = eng.badge_pooled_embedding(lg.cuda(), em.cuda(), 128).cpu()
    ref = O.gradient_embeddings(lg, em, 128, use_adaptive_pool=True)
    assert got.shape == (300, 512)
    assert torch.allclose(got, ref, rtol=1e-4, atol=1e-8)


def test_row_norms(eng):
    rng = np.random.default_rng(4)
    xi = torch.from_numpy(rng.integers(-1, 2, size=(1000, 2048)).astype(np.float32))
    assert torch.equal(eng.row_norm2(xi.cuda()).cpu(), xi.square().sum(1))
    xf = torch.randn(777, 36)
    assert torch.allclose(eng.row_norm2(xf.cuda()).cpu(), xf.square().sum(1), rtol=1e-5)


def test_full_size_margin_properties(eng):
    """BASELINE config 1 shape (80k x 1000, B = 10k): sortedness + subsample vs oracle."""
    torch.manual_seed(0)
    logits = torch.randn(80000, 1000, device="cuda") * 3
    scores = eng.score_softmax(logits, O.MODE_MARGIN)
    pos = eng.select_smallest(scores, 10000).cpu().numpy()
    s = scores.cpu().numpy()
    assert len(set(pos.tolist())) == 10000
    key = s[pos].astype(np.float64) * 1e6 + 0
    assert np.all(np.diff(s[pos]) >= 0)
    ties = np.diff(s[pos]) == 0
    assert np.all(np.diff(pos)[ties] > 0)                        # ties by position
    rest = np.ones(80000, dtype=bool)
    rest[pos] = False
    assert s[rest].min() >= s[pos].max()
    sub = np.random.default_rng(0).choice(80000, 2000, replace=False)
    ref = O.softmax_scores(logits[torch.from_numpy(sub).cuda()].cpu(), O.MODE_MARGIN).numpy()
    np.testing.assert_allclose(s[sub], ref, rtol=0, atol=TOL_PROB)


def test_topb_pack_merge_equals_global_select(eng):
    """The multi-GPU merge primitive without the all-gather: shard a score vector in 3, pack each
    shard's local top-B, merge the packed words -> the single-GPU K1b result (ties included)."""
    rng = np.random.default_rng(11)
    n, b = 90000, 7000
    scores = torch.from_numpy((rng.integers(0, 400, size=n) / 128.0).astype(np.float32)).cuda()
    bounds = [0, 30000, 61000, n]
    words = []
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        loc = scores[lo:hi].contiguous()
        pos = eng.select_smallest(loc, min(b, hi - lo))
        words.append(eng.topb_pack(loc, pos, lo, b))
    ref = eng.select_smallest(scores, b).cpu().numpy()
    assert np.array_equal(eng.topb_merge(torch.cat(words), b).cpu().numpy(), ref)
    assert np.array_equal(eng.topb_merge(torch.cat(words), b, list_len=b).cpu().numpy(), ref)


@pytest.mark.parametrize("n,c", [(5003, 1000), (4097, 2048), (9000, 64), (70001, 4), (6000, 1024)])
def test_pipelined_rows_kernels_equal_direct_kernels(eng, n, c):
    """K1/K2 TMA bulk-copy pipeline (n >= 4096, contiguous rows) vs the direct-load kernels, which take rows with a
    leading dimension ld != c: the same logits once contiguous and once in an [n, c + 4] buffer (NaN padding) sliced to
    c columns.  Same row code, so scores and BADGE factors must be bit-identical; and both match the oracle."""
    torch.manual_seed(n + c)
    logits = torch.randn(n, c) * 3
    dense = logits.cuda()
    padded = torch.full((n, c + 4), float("nan"), device="cuda")
    padded[:, :c] = dense
    strided = padded[:, :c]
    assert strided.stride(0) == c + 4
    res = {}
    for name, dev in (("direct", strided), ("pipelined", dense)):
        res[name] = [eng.score_softmax(dev, m).cpu() for m in (0, 1, 2)] + \
            [t.cpu() for t in eng.badge_factors(dev, 128)]
    for a, b in zip(res["direct"], res["pipelined"]):
        assert torch.equal(a, b)
    assert torch.allclose(res["pipelined"][0], O.softmax_scores(logits, O.MODE_MARGIN), rtol=0, atol=TOL_PROB)
    assert torch.allclose(res["pipelined"][3][:, :c], O.badge_factors(logits, 128), rtol=0, atol=1e-7)


@pytest.mark.parametrize("n,c,b", FUSED_TAIL_SHAPES)
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_fused_tail_equals_score_then_select(eng, n, c, b, mode):
    """alq_uncertainty_tail (K1 + K1b as one launch: per-CTA key lists, two global 11-bit histogram levels, winners
    ordered either through per-CTA score buckets or by ranking against the whole list) against the two separate kernels:
    identical scores, identical ordered positions, on both routes."""
    logits = fused_tail_logits(n, c, b, mode)
    ref_s = eng.score_softmax(logits, mode)
    ref_p = eng.select_smallest(ref_s, b)
    try:
        for buckets in (1, 0):
            eng.set_option("tail_buckets", buckets)
            s, p = eng.uncertainty_tail(logits, mode, b)
            assert torch.equal(s, ref_s)
            assert torch.equal(p, ref_p), buckets
    finally:
        eng.set_option("tail_buckets", 1)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_fused_tail_with_skewed_scores(eng, mode):
    """Scores that do not spread evenly between the candidate range's edges (per-row temperature over five decades: the
    margins pile up next to 0, the confidences next to 1/C and 1): the score buckets are uneven, and with the 40-row pool
    piled into a few of them one bucket exceeds its capacity and the launch falls back to the general route by itself."""
    for logits, b in skewed_tail_pools(mode):
        ref_s = eng.score_softmax(logits, mode)
        s, p = eng.uncertainty_tail(logits, mode, b)
        assert torch.equal(s, ref_s)
        assert torch.equal(p, eng.select_smallest(ref_s, b))


def test_fused_tail_with_massive_ties(eng):
    """Dyadic logits: thousands of rows share a score exactly, the threshold bin of the fused selection holds far more
    keys than the budget needs (and more than one shared-memory chunk): ties must still resolve by position."""
    for logits, b in tied_tail_pools():
        for mode in (0, 1, 2):
            ref_s = eng.score_softmax(logits, mode)
            s, p = eng.uncertainty_tail(logits, mode, b)
            assert torch.equal(s, ref_s)
            assert torch.equal(p, eng.select_smallest(ref_s, b))
            assert np.array_equal(p.cpu().numpy(), O.select_smallest(ref_s.cpu(), b))
    const = torch.zeros(70000, 16, device="cuda")            # every score identical: the first b positions, in order
    s, p = eng.uncertainty_tail(const, 0, 5000)
    assert p.cpu().tolist() == list(range(5000))


def test_full_size_ordered_list_against_the_oracle_with_near_tie_certificate(eng):
    """BASELINE config 1 at full size, the ORDERED 10 000-row list against the oracle (torch-CPU softmax in loader
    batches of 128 + stable sort, margin_sampler.py:33-42), Margin and Confidence.  K1 evaluates exp through ex2.approx,
    so a score may differ from torch's in the last bits and two rows whose oracle scores are closer than that may
    swap places.  Certificate: walking both lists position by position, the oracle scores of the two rows at the same
    rank never differ by more than the stated per-sample tolerance, and the selected SETS differ only by rows whose
    oracle score is within that tolerance of the budget boundary."""
    torch.manual_seed(0)
    logits = torch.randn(80000, 1000) * 3
    dev = logits.cuda()
    for mode in (O.MODE_MARGIN, O.MODE_LEAST_CONFIDENCE):
        ref_scores = O.softmax_scores(logits, mode)
        ref = O.select_smallest(ref_scores, 10000)
        got_scores, got = eng.uncertainty_tail(dev, mode, 10000)
        got = got.cpu().numpy()
        rs = ref_scores.numpy()
        assert np.abs(got_scores.cpu().numpy() - rs).max() <= TOL_PROB
        assert np.abs(rs[got] - rs[ref]).max() <= 2 * TOL_PROB                      # same score sequence up to the tolerance
        boundary = rs[ref[-1]]
        diff = np.setxor1d(got, ref)
        assert len(diff) < 200 and (len(diff) == 0 or np.abs(rs[diff] - boundary).max() <= 2 * TOL_PROB)
