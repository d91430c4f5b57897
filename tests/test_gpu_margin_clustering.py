"""K7 / K8 / MarginClusteringSampler on the H100: distances and merge lists bit for bit against the NumPy twin
(tests/ward_oracle.py, itself checked against scipy on the CPU tier), labels against sklearn's golden labels, picks
against the reference's golden picks in both rounds, int64 addressing past 2^31 entries, and the memory guard."""
import os

import numpy as np
import pytest
import torch

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


@pytest.mark.parametrize("n", [2, 3, 63, 65, 1000])
@pytest.mark.parametrize("d", [1, 7, 64, 2048])
def test_k7_is_scipys_pdist_bit_for_bit(eng, n, d):
    x = _rows(n, d, n * 7 + d)
    got = eng.pdist(torch.from_numpy(x).cuda()).cpu().numpy()
    assert np.array_equal(got, W.pdist_square(x))


def test_k7_strided_input_and_zero_pad_columns(eng):
    x = _rows(130, 37, 1)
    want = W.pdist_square(x)
    big = torch.zeros((130, 53), device="cuda")
    big[:, :37] = torch.from_numpy(x).cuda()
    strided = big[:, :37]                                  # ld 53, unaligned rows
    assert strided.stride(0) == 53
    assert np.array_equal(eng.pdist(strided).cpu().numpy(), want)
    padded = torch.zeros((130, 40), device="cuda")         # the 16-byte row padding of the pool forward
    padded[:, :37] = torch.from_numpy(x).cuda()
    assert np.array_equal(eng.pdist(padded).cpu().numpy(), want)
    out = torch.full((140, 150), -1.0, dtype=torch.float64, device="cuda")   # ldd > n: the rest is untouched
    eng.pdist(padded, out=out)
    assert np.array_equal(out[:130, :130].cpu().numpy(), want) and bool((out[130:] == -1).all())


def _chain_cases():
    rng = np.random.default_rng(2)
    yield "float", _rows(1500, 64, 3)
    base = rng.integers(0, 3, size=(150, 4))
    yield "int_ties", base[rng.integers(0, 150, size=1200)].astype(np.float32)
    yield "line5000", W.shrinking_gap_line(5000)
    yield "n2", _rows(2, 5, 4)


@pytest.mark.parametrize("name", [c[0] for c in _chain_cases()])
def test_k8_merge_list_is_the_oracles_bit_for_bit(eng, name):
    x = dict(_chain_cases())[name]
    D = W.pdist_square(x)
    xy_w, md_w, longest = W.ward_nn_chain(D)
    if name == "line5000":
        assert longest == 5000
    dist = torch.from_numpy(D).cuda()
    xy, md = eng.nn_chain(dist)
    assert np.array_equal(xy.cpu().numpy(), xy_w) and np.array_equal(md.cpu().numpy(), md_w)


def test_k8_at_12000_rows_of_2048(eng):
    x = torch.from_numpy(_rows(12000, 2048, 9)).cuda()
    dist = eng.pdist(x)
    D = dist.cpu().numpy()                                 # K7 is checked bit for bit above; K8 consumes dist
    xy, md = eng.nn_chain(dist)
    xy_w, md_w, _ = W.ward_nn_chain(D)
    assert np.array_equal(xy.cpu().numpy(), xy_w) and np.array_equal(md.cpu().numpy(), md_w)


def test_ward_labels_equal_sklearns_golden_labels(eng, gold):
    for tag in "fstb":
        for h in range(int(gold[f"{tag}_hac_calls"])):
            got = eng.ward_labels(torch.from_numpy(gold[f"{tag}_hac{h}_x"]).cuda(), 20)
            assert np.array_equal(got, gold[f"{tag}_hac{h}_labels"]), (tag, h)


@pytest.mark.parametrize("tag", ["f", "s", "t", "b"])
def test_sampler_returns_the_reference_picks_in_both_rounds(eng, gold, tag):
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


def test_int64_addressing_at_46500_rows(eng):
    """n^2 = 2.16e9 > 2^31 entries (17.3 GB): sampled K7 entries of the last rows against NumPy fp64, and 20
    well-separated integer blobs that the 20-cluster cut must return as they were built."""
    from active_learning_b200.engine import ward_labels_host
    n, blobs = 46500, 20
    rng = np.random.default_rng(46500)
    blob = np.repeat(np.arange(blobs), n // blobs)
    x = rng.integers(0, 8, size=(n, 4)).astype(np.float32)
    x[:, 0] += blob * 10000.0
    perm = rng.permutation(n)
    x, blob = x[perm], blob[perm]
    xd = torch.from_numpy(x).cuda()
    dist = eng.pdist(xd)
    i = np.concatenate([np.full(64, n - 1), np.full(64, n - 2), rng.integers(46341, n, 128)])
    j = rng.integers(0, n, len(i))
    got = dist[torch.from_numpy(i).cuda(), torch.from_numpy(j).cuda()].cpu().numpy()
    got_t = dist[torch.from_numpy(j).cuda(), torch.from_numpy(i).cuda()].cpu().numpy()
    diff = x[i].astype(np.float64) - x[j].astype(np.float64)
    want = np.sqrt(np.cumsum(diff * diff, axis=1)[:, -1])
    assert np.array_equal(got, want) and np.array_equal(got_t, want)
    xy, md = eng.nn_chain(dist)
    del dist
    labels = ward_labels_host(xy.cpu().numpy(), md.cpu().numpy(), n, blobs)
    # same partition as the construction: every blob is one cluster and the 20 clusters are distinct
    pairs = set(zip(blob.tolist(), labels.tolist()))
    assert len(pairs) == blobs and len({b for b, _ in pairs}) == blobs and len({lab for _, lab in pairs}) == blobs


def test_memory_guard_raises_before_allocating(eng):
    from active_learning_b200._lib import AlqError
    n = 200000                                            # 8 n^2 = 320 GB
    x = torch.rand((n, 4), device="cuda")
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    with pytest.raises(AlqError, match=f"n={n}"):
        eng.ward_labels(x, 20)
    assert torch.cuda.max_memory_allocated() - before < (16 << 20)      # nothing of the matrix's 8 n^2 scale


def test_value_errors_as_sklearn_raises(eng):
    with pytest.raises(ValueError):
        eng.ward_labels(torch.rand((19, 8), device="cuda"), 20)
    x = torch.rand((40, 8), device="cuda")
    x[3, 2] = float("inf")
    with pytest.raises(ValueError):
        eng.ward_labels(x, 20)


def test_k8_non_finite_row_is_a_numeric_error_and_the_context_stays_usable(eng):
    """A matrix with no finite distance from row 0: the first scan of the chain finds no candidate, every CTA leaves
    the walk together and the call reports ALQ_ERR_NUMERIC.  The next call on the same context is unaffected."""
    from active_learning_b200._lib import AlqError
    x = _rows(40, 6, 40)
    D = W.pdist_square(x)
    bad = D.copy()
    bad[0, :] = np.inf
    bad[:, 0] = np.inf
    with pytest.raises(AlqError, match="ALQ_ERR_NUMERIC"):
        eng.nn_chain(torch.from_numpy(bad).cuda())
    xy_w, md_w, _ = W.ward_nn_chain(D)
    xy, md = eng.nn_chain(torch.from_numpy(D).cuda())
    assert np.array_equal(xy.cpu().numpy(), xy_w) and np.array_equal(md.cpu().numpy(), md_w)


def test_nn_chain_and_ward_tree_validate_their_inputs(eng):
    from active_learning_b200._lib import AlqError
    D = torch.from_numpy(W.pdist_square(_rows(30, 4, 30))).cuda()
    with pytest.raises(AlqError):
        eng.nn_chain(D.float())                            # 4-byte entries: K8 would read past the matrix
    with pytest.raises(AlqError):
        eng.nn_chain(D, n=31)                              # n larger than the matrix
    with pytest.raises(AlqError):
        eng.nn_chain(D.t()[:, :30].contiguous().t())       # column-major
    with pytest.raises(AlqError):
        eng.nn_chain(D.cpu())
    x = torch.rand((30, 4), device="cuda")
    x[7, 1] = float("nan")
    with pytest.raises(ValueError):
        eng.ward_tree(x)


def test_ward_tree_returns_the_matrix_to_the_device(eng):
    n = 3000                                               # 72 MB of fp64 matrix
    x = torch.from_numpy(_rows(n, 16, 3000)).cuda()
    torch.cuda.synchronize()
    before = torch.cuda.memory_reserved()
    eng.ward_labels(x, 20)
    assert torch.cuda.memory_reserved() < before + 8 * n * n

