"""K7 / K8 over scipy's condensed distance vector on the H100: distances bit for bit against scipy's pdist, merge lists
bit for bit against the NumPy twin (tests/ward_oracle.py) and against the square layout, int64 offsets past 2^31 and
2^32 entries, the numeric error, argument checks, and the automatic layout choice through the product path."""
import ctypes
import os

import numpy as np
import pytest
import torch
from scipy.spatial.distance import pdist as scipy_pdist

import ward_oracle as W

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def eng():
    from active_learning_b200.engine import Engine
    return Engine()


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(os.path.join(HERE, "golden", "reference_golden_margin_clustering.npz")))


def _rows(n, d, seed):
    rng = np.random.default_rng(seed)
    return np.maximum(rng.standard_normal((n, d)), 0).astype(np.float32)


def _condensed(D):
    return np.ascontiguousarray(D[np.triu_indices(D.shape[0], 1)])


def _cidx(i, j, n):
    i, j = np.asarray(i, dtype=np.int64), np.asarray(j, dtype=np.int64)
    return n * i - i * (i + 1) // 2 + (j - i - 1)


@pytest.mark.parametrize("n", [2, 3, 63, 65, 1000])
@pytest.mark.parametrize("d", [1, 7, 64, 2048])
def test_condensed_k7_is_scipys_pdist_bit_for_bit(eng, n, d):
    x = _rows(n, d, n * 7 + d)
    got = eng.pdist(torch.from_numpy(x).cuda(), condensed=True)
    assert got.dim() == 1 and got.shape[0] == n * (n - 1) // 2
    assert np.array_equal(got.cpu().numpy(), scipy_pdist(x.astype(np.float64)))


def test_condensed_k7_strided_input_zero_pad_columns_and_a_longer_buffer(eng):
    x = _rows(130, 37, 1)
    want = scipy_pdist(x.astype(np.float64))
    big = torch.zeros((130, 53), device="cuda")
    big[:, :37] = torch.from_numpy(x).cuda()
    strided = big[:, :37]                                  # ld 53, unaligned rows
    assert strided.stride(0) == 53
    assert np.array_equal(eng.pdist(strided, condensed=True).cpu().numpy(), want)
    padded = torch.zeros((130, 40), device="cuda")         # the 16-byte row padding of the pool forward
    padded[:, :37] = torch.from_numpy(x).cuda()
    assert np.array_equal(eng.pdist(padded, condensed=True).cpu().numpy(), want)
    m = len(want)
    out = torch.full((m + 777,), -1.0, dtype=torch.float64, device="cuda")
    assert eng.pdist(padded, out=out, condensed=True) is out
    assert np.array_equal(out[:m].cpu().numpy(), want) and bool((out[m:] == -1).all())


def _chain_cases():
    rng = np.random.default_rng(2)
    yield "float", _rows(1500, 64, 3)
    base = rng.integers(0, 3, size=(150, 4))
    yield "int_ties", base[rng.integers(0, 150, size=1200)].astype(np.float32)
    yield "line5000", W.shrinking_gap_line(5000)
    yield "n2", _rows(2, 5, 4)


@pytest.mark.parametrize("name", [c[0] for c in _chain_cases()])
def test_condensed_k8_merge_list_is_the_oracles_bit_for_bit(eng, name):
    x = dict(_chain_cases())[name]
    D = W.pdist_square(x)
    xy_w, md_w, longest = W.ward_nn_chain(D)
    if name == "line5000":
        assert longest == 5000
    xy, md = eng.nn_chain(torch.from_numpy(_condensed(D)).cuda())
    assert np.array_equal(xy.cpu().numpy(), xy_w) and np.array_equal(md.cpu().numpy(), md_w)


def _both_layouts(eng, x):
    """K7 + K8 in the square layout, then (the matrix freed) in the condensed one, on the same rows."""
    out = []
    for condensed in (False, True):
        dist = eng.pdist(x, condensed=condensed)
        xy, md = eng.nn_chain(dist)
        out.append((xy.cpu().numpy(), md.cpu().numpy()))
        del dist, xy, md
        torch.cuda.empty_cache()
    return out


def test_condensed_k8_equals_the_square_layout_at_12000_rows_of_2048(eng):
    (xy_s, md_s), (xy_c, md_c) = _both_layouts(eng, torch.from_numpy(_rows(12000, 2048, 9)).cuda())
    assert np.array_equal(xy_c, xy_s) and np.array_equal(md_c, md_s)


def test_both_layouts_past_2_31_entries_at_70000_rows(eng):
    """n (n - 1) / 2 = 2.45e9 > 2^31 condensed entries (19.6 GB); the square matrix is 39.2 GB."""
    n = 70000
    if eng._ward_free_bytes() < eng.ward_bytes(n):
        pytest.skip(f"the square layout at n={n} needs {eng.ward_bytes(n)} bytes of free device memory")
    (xy_s, md_s), (xy_c, md_c) = _both_layouts(eng, torch.from_numpy(_rows(n, 64, 70000)).cuda())
    assert np.array_equal(xy_c, xy_s) and np.array_equal(md_c, md_s)


def test_ward_labels_past_2_32_entries_take_the_condensed_layout(eng, monkeypatch):
    """110 000 rows: 6.05e9 > 2^32 condensed entries (48.4 GB) where the square matrix (96.8 GB) cannot fit an 80 GB
    card.  Sampled K7 entries of the last rows against NumPy fp64 (read before K8 consumes the vector), and 20
    well-separated integer blobs that the 20-cluster cut must return as they were built."""
    n, blobs = 110000, 20
    free = eng._ward_free_bytes()                          # what ward_tree's own choice sees
    if free < eng.ward_condensed_bytes(n):
        pytest.skip(f"the condensed layout at n={n} needs {eng.ward_condensed_bytes(n)} bytes, {free} are free")
    rng = np.random.default_rng(110000)
    blob = np.repeat(np.arange(blobs), n // blobs)
    x = rng.integers(0, 8, size=(n, 4)).astype(np.float32)
    x[:, 0] += blob * 10000.0
    perm = rng.permutation(n)
    x, blob = x[perm], blob[perm]
    i = np.concatenate([np.full(64, n - 2), np.full(64, n - 3), rng.integers(93000, n - 1, 128)])
    j = i + 1 + rng.integers(0, n - 1 - i)                 # i < j < n
    j[0] = n - 1                                           # the vector's last entry
    idx = _cidx(i, j, n)
    assert (idx >= 1 << 32).all() and idx.max() == n * (n - 1) // 2 - 1
    sampled = {}
    real_pdist = eng.pdist

    def pdist(xx, out=None, condensed=False):
        dist = real_pdist(xx, out=out, condensed=condensed)
        sampled["condensed"] = condensed
        sampled["got"] = dist[torch.from_numpy(idx).cuda()].cpu().numpy()
        return dist

    monkeypatch.setattr(eng, "pdist", pdist)
    labels = eng.ward_labels(torch.from_numpy(x).cuda(), blobs)
    assert sampled["condensed"] is True
    diff = x[i].astype(np.float64) - x[j].astype(np.float64)
    want = np.sqrt(np.cumsum(diff * diff, axis=1)[:, -1])
    assert np.array_equal(sampled["got"], want)
    pairs = set(zip(blob.tolist(), labels.tolist()))
    assert len(pairs) == blobs and len({b for b, _ in pairs}) == blobs and len({lab for _, lab in pairs}) == blobs


def test_condensed_k8_non_finite_row_is_a_numeric_error_and_the_context_stays_usable(eng):
    from active_learning_b200._lib import AlqError
    x = _rows(40, 6, 40)
    D = W.pdist_square(x)
    bad = D.copy()
    bad[0, :] = np.inf
    bad[:, 0] = np.inf
    with pytest.raises(AlqError, match="ALQ_ERR_NUMERIC"):
        eng.nn_chain(torch.from_numpy(_condensed(bad)).cuda())
    xy_w, md_w, _ = W.ward_nn_chain(D)
    xy, md = eng.nn_chain(torch.from_numpy(_condensed(D)).cuda())
    assert np.array_equal(xy.cpu().numpy(), xy_w) and np.array_equal(md.cpu().numpy(), md_w)


def test_condensed_entry_points_and_nn_chain_validate_their_inputs(eng):
    from active_learning_b200._lib import AlqError
    D = torch.from_numpy(_condensed(W.pdist_square(_rows(30, 4, 30)))).cuda()      # 435 entries
    for bad in (torch.cat([D, D[:1]]), D[:-1], D[:0], D.float(), D.cpu()):
        with pytest.raises(AlqError):
            eng.nn_chain(bad)
    with pytest.raises(AlqError):
        eng.nn_chain(D, n=31)                              # n must match the length
    with pytest.raises(AlqError):
        eng.nn_chain(torch.cat([D, D])[::2])               # not contiguous
    x = torch.rand((30, 4), device="cuda")
    for out in (torch.empty(434, dtype=torch.float64, device="cuda"), torch.empty(435, device="cuda"),
                torch.empty(435, dtype=torch.float64), torch.empty((435, 1), dtype=torch.float64, device="cuda")):
        with pytest.raises(AlqError):
            eng.pdist(x, out=out, condensed=True)
    lib, h, null, s = eng.lib, eng._h, ctypes.c_void_p(0), eng._stream()
    p = ctypes.c_void_p(D.data_ptr())
    xp = ctypes.c_void_p(x.data_ptr())
    xy = torch.empty((29, 2), dtype=torch.int32, device="cuda")
    md = torch.empty(29, dtype=torch.float64, device="cuda")
    xyp, mdp = ctypes.c_void_p(xy.data_ptr()), ctypes.c_void_p(md.data_ptr())
    invalid = 1
    assert lib.alq_pdist_f64_condensed(None, xp, 30, 4, 4, p, s) == invalid
    assert lib.alq_pdist_f64_condensed(h, null, 30, 4, 4, p, s) == invalid
    assert lib.alq_pdist_f64_condensed(h, xp, 30, 4, 4, null, s) == invalid
    assert lib.alq_pdist_f64_condensed(h, xp, 0, 4, 4, p, s) == invalid
    assert lib.alq_pdist_f64_condensed(h, xp, 30, 0, 4, p, s) == invalid
    assert lib.alq_pdist_f64_condensed(h, xp, 30, 4, 3, p, s) == invalid
    assert lib.alq_pdist_f64_condensed(h, xp, 65535 * 64 + 1, 4, 4, p, s) == invalid
    assert lib.alq_ward_nn_chain_condensed(None, p, 30, xyp, mdp, s) == invalid
    assert lib.alq_ward_nn_chain_condensed(h, null, 30, xyp, mdp, s) == invalid
    assert lib.alq_ward_nn_chain_condensed(h, p, 30, null, mdp, s) == invalid
    assert lib.alq_ward_nn_chain_condensed(h, p, 30, xyp, null, s) == invalid
    assert lib.alq_ward_nn_chain_condensed(h, p, 1, xyp, mdp, s) == invalid
    assert lib.alq_ward_nn_chain_condensed(h, p, 1 << 31, xyp, mdp, s) == invalid
    torch.cuda.synchronize()
    xy_w, md_w, _ = W.ward_nn_chain(W.pdist_square(_rows(30, 4, 30)))   # the context is still usable
    xy, md = eng.nn_chain(D)
    assert np.array_equal(xy.cpu().numpy(), xy_w) and np.array_equal(md.cpu().numpy(), md_w)


@pytest.fixture
def square_does_not_fit(eng, monkeypatch):
    """The free-bytes probe reports exactly the condensed layout's need for each query's n, so only it fits; records
    which layouts K7 was asked for."""
    layouts = []
    real_tree, real_pdist = eng.ward_tree, eng.pdist

    def ward_tree(x):
        need = eng.ward_condensed_bytes(x.shape[0])
        assert need < eng.ward_bytes(x.shape[0])
        monkeypatch.setattr(eng, "_ward_free_bytes", lambda: need)
        return real_tree(x)

    def pdist(x, out=None, condensed=False):
        layouts.append(condensed)
        return real_pdist(x, out=out, condensed=condensed)

    monkeypatch.setattr(eng, "ward_tree", ward_tree)
    monkeypatch.setattr(eng, "pdist", pdist)
    return layouts


def test_ward_labels_equal_sklearns_golden_labels_in_the_condensed_layout(eng, gold, square_does_not_fit):
    for tag in "fstb":
        for h in range(int(gold[f"{tag}_hac_calls"])):
            got = eng.ward_labels(torch.from_numpy(gold[f"{tag}_hac{h}_x"]).cuda(), 20)
            assert np.array_equal(got, gold[f"{tag}_hac{h}_labels"]), (tag, h)
    assert square_does_not_fit and all(square_does_not_fit)


@pytest.mark.parametrize("tag", ["f", "s", "t", "b"])
def test_sampler_returns_the_reference_picks_in_the_condensed_layout(eng, gold, tag, square_does_not_fit):
    from helpers import HeadNet, make_strategy
    emb = torch.from_numpy(gold[f"{tag}_emb"])
    kw = {}
    if int(gold[f"{tag}_subset"]) >= 0:
        kw["subset_unlabeled"] = int(gold[f"{tag}_subset"])
    if f"{tag}_logits" in gold:
        logits, net = torch.from_numpy(gold[f"{tag}_logits"]), None
    else:
        logits, net = None, HeadNet(emb, torch.from_numpy(gold[f"{tag}_weight"]), torch.from_numpy(gold[f"{tag}_bias"]))
    s = make_strategy("MarginClusteringSampler", logits, emb, gold[f"{tag}_eval"], gold[f"{tag}_labeled"],
                      int(gold[f"{tag}_bs"]), engine=eng, net=net, **kw)
    for r in range(2):
        np.random.seed(100 + r)
        idx, cost = s.query(float(gold[f"{tag}_budget"]))
        assert [int(i) for i in idx] == gold[f"{tag}_r{r}_picks"].tolist(), (tag, r)
        assert cost == int(gold[f"{tag}_r{r}_cost"])
        s.update(idx, cost)
    assert square_does_not_fit and all(square_does_not_fit)


def test_condensed_ward_tree_returns_the_vector_to_the_device(eng, square_does_not_fit):
    n = 3000
    x = torch.from_numpy(_rows(n, 16, 3000)).cuda()
    torch.cuda.synchronize()
    before = torch.cuda.memory_reserved()
    eng.ward_labels(x, 20)
    assert square_does_not_fit == [True]
    assert torch.cuda.memory_reserved() < before + 4 * n * (n - 1)
