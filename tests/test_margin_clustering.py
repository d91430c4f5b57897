"""MarginClusteringSampler without a GPU: the NumPy twin of K7/K8 against scipy's Ward tree (bit for bit), the host
helper alq_ward_labels (through ctypes, no device) against sklearn and the twin, the round robin against its loop form,
and the sampler's host logic replaying the reference's goldens (tests/golden/make_golden_margin_clustering.py) with
the twin injected as the engine."""
import ctypes
import os

import numpy as np
import pytest
import torch

import ward_oracle as W
from helpers import HeadNet, OracleEngine, make_strategy

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(os.path.join(HERE, "golden", "reference_golden_margin_clustering.npz")))


def _fixtures():
    rng = np.random.default_rng(11)
    yield "relu", np.maximum(rng.standard_normal((500, 40)), 0).astype(np.float32)
    base = rng.integers(0, 3, size=(60, 5))
    yield "ties", base[rng.integers(0, 60, size=400)].astype(np.float32)
    yield "line", W.shrinking_gap_line(400)


class WardOracleEngine(OracleEngine):
    """The CPU engine stub with the Ward path of the twin."""

    def ward_labels(self, x, n_clusters):
        return W.ward_labels(x.numpy(), n_clusters)


def _host_labels(xy, md, n, k):
    from active_learning_b200 import _lib, build
    if not os.path.exists(_lib.LIB_PATH):
        build.build()
    lib = _lib.load()
    xy = np.ascontiguousarray(xy, dtype=np.int32)
    md = np.ascontiguousarray(md, dtype=np.float64)
    out = np.full(n, -1, dtype=np.int32)
    rc = lib.alq_ward_labels(ctypes.c_void_p(xy.ctypes.data), ctypes.c_void_p(md.ctypes.data), n, k,
                             ctypes.c_void_p(out.ctypes.data))
    return rc, out


@pytest.mark.parametrize("name,x", list(_fixtures()), ids=[f[0] for f in _fixtures()])
def test_oracle_nn_chain_is_scipys_ward_tree_bit_for_bit(name, x):
    hierarchy = pytest.importorskip("scipy.cluster.hierarchy")
    from scipy.spatial.distance import pdist, squareform
    D = W.pdist_square(x)
    assert np.array_equal(D, squareform(pdist(x, "euclidean")))
    xy, md, longest = W.ward_nn_chain(D)
    assert (xy[:, 0] < xy[:, 1]).all()
    Z = W.linkage_from_merges(xy, md, len(x))
    assert np.array_equal(Z, hierarchy.ward(x))          # all four columns
    if name == "line":
        assert longest == len(x)                          # the chain walks the whole line before its first merge


def test_host_labels_equal_sklearn_and_the_oracle_cut():
    cluster = pytest.importorskip("sklearn.cluster")
    for _name, x in _fixtures():
        xy, md, _ = W.ward_nn_chain(W.pdist_square(x))
        Z = W.linkage_from_merges(xy, md, len(x))
        for k in (1, 2, 20, 33):
            rc, got = _host_labels(xy, md, len(x), k)
            assert rc == 0
            want = cluster.AgglomerativeClustering(n_clusters=k).fit(x).labels_
            assert np.array_equal(got, want)
            assert np.array_equal(got, W.hc_cut(k, Z[:, :2].astype(np.int64), len(x)))


def test_host_labels_on_random_trees_match_the_oracle_cut():
    """Arbitrary valid merge lists (random and heavily tied distances), no sklearn needed."""
    rng = np.random.default_rng(5)
    for trial in range(30):
        n = int(rng.integers(2, 300))
        live = list(range(n))
        xy = np.empty((n - 1, 2), dtype=np.int64)
        for k in range(n - 1):
            a, b = sorted(rng.choice(len(live), 2, replace=False))
            xy[k] = (live[a], live[b])
            del live[a]                                   # the merged cluster keeps the larger index
        md = rng.integers(0, 4, n - 1).astype(np.float64) if trial % 2 else rng.random(n - 1)
        Z = W.linkage_from_merges(xy, md, n)
        for k in sorted({1, min(n, 2), min(n, 20), n}):
            rc, got = _host_labels(xy, md, n, k)
            assert rc == 0 and np.array_equal(got, W.hc_cut(k, Z[:, :2].astype(np.int64), n))


def test_host_labels_reject_more_clusters_than_rows_and_bad_lists():
    xy = np.array([[0, 1], [1, 2]])
    md = np.array([1.0, 2.0])
    assert _host_labels(xy, md, 3, 4)[0] != 0
    assert _host_labels(np.array([[0, 5], [1, 2]]), md, 3, 2)[0] != 0
    # a pair whose clusters are already joined: row 2 is never merged, so its label would go unwritten
    assert _host_labels(np.array([[0, 1], [0, 1]]), md, 3, 2)[0] != 0
    assert _host_labels(np.array([[0, 1], [1, 0]]), md, 3, 1)[0] != 0
    assert _host_labels(np.array([[0, 2], [0, 1]]), md, 3, 2)[0] == 0      # any order of a spanning tree is valid
    assert _host_labels(xy, md, 3, 3)[0] == 0
    from active_learning_b200.engine import ward_labels_host
    with pytest.raises(ValueError):
        ward_labels_host(xy, md, 3, 4)


def test_round_robin_equals_the_pass_loop():
    from active_learning_b200.query_strategies.margin_clustering import round_robin
    rng = np.random.default_rng(3)
    for trial in range(40):
        n = int(rng.integers(1, 400))
        assignment = rng.integers(0, int(rng.integers(1, 25)), n)
        margins = (rng.integers(0, 5, n) / 4.0 if trial % 3 == 0 else rng.random(n)).astype(np.float32)
        for budget in (0, 1, 7, n // 2, n, n + 5):
            p1, left1 = round_robin(assignment, margins, budget)
            p2, left2 = W.round_robin(assignment, margins, budget)
            assert p1.tolist() == p2.tolist() and np.array_equal(left1, left2)


def _sampler(gold, tag, engine):
    emb = torch.from_numpy(gold[f"{tag}_emb"])
    kw = {}
    if int(gold[f"{tag}_subset"]) >= 0:
        kw["subset_unlabeled"] = int(gold[f"{tag}_subset"])
    if f"{tag}_logits" in gold:
        logits, net = torch.from_numpy(gold[f"{tag}_logits"]), None
    else:
        logits, net = None, HeadNet(emb, torch.from_numpy(gold[f"{tag}_weight"]), torch.from_numpy(gold[f"{tag}_bias"]))
    return make_strategy("MarginClusteringSampler", logits, emb, gold[f"{tag}_eval"], gold[f"{tag}_labeled"],
                         int(gold[f"{tag}_bs"]), engine=engine, net=net, **kw)


@pytest.mark.parametrize("tag", ["f", "s", "t", "b"])
def test_oracle_sampler_replays_the_reference_goldens(gold, tag):
    s = _sampler(gold, tag, WardOracleEngine())
    for r in range(2):
        np.random.seed(100 + r)
        idx, cost = s.query(float(gold[f"{tag}_budget"]))
        assert [int(i) for i in idx] == gold[f"{tag}_r{r}_picks"].tolist()
        assert cost == int(gold[f"{tag}_r{r}_cost"]) and all(isinstance(i, np.int64) for i in idx)
        assert not s.feature_net.training                 # left in eval(), as the reference leaves it
        s.update(idx, cost)


def test_oracle_labels_replay_sklearns_golden_labels(gold):
    for tag in "fstb":
        for h in range(int(gold[f"{tag}_hac_calls"])):
            assert np.array_equal(W.ward_labels(gold[f"{tag}_hac{h}_x"]), gold[f"{tag}_hac{h}_labels"])


def test_reuse_runs_no_clustering_and_subset_clusters_every_round(gold):
    calls = []

    class Counting(WardOracleEngine):
        def ward_labels(self, x, n_clusters):
            calls.append(x.shape[0])
            return super().ward_labels(x, n_clusters)

    for tag, want in (("f", 1), ("s", 2)):
        calls.clear()
        s = _sampler(gold, tag, Counting())
        for r in range(2):
            np.random.seed(100 + r)
            idx, cost = s.query(float(gold[f"{tag}_budget"]))
            s.update(idx, cost)
        assert len(calls) == want


def test_too_few_rows_and_non_finite_rows_raise_value_error():
    with pytest.raises(ValueError):
        W.ward_labels(np.zeros((19, 3), dtype=np.float32))
    x = np.ones((30, 3), dtype=np.float32)
    x[4, 1] = np.nan
    with pytest.raises(ValueError):
        W.ward_labels(x)


def test_sharded_group_is_refused(gold):
    from active_learning_b200._lib import AlqError

    class Group:
        world_size = 2

    s = _sampler(gold, "f", WardOracleEngine())
    s._shard_group = Group()
    with pytest.raises(AlqError, match="one GPU"):
        s.query(10.0)


def test_dispatch_and_drop_in_binding():
    from active_learning_b200.integration import make_drop_in
    from active_learning_b200.query_strategies.get_strategy import ACCELERATED, NOT_ON_THIS_PATH, get_strategy
    from active_learning_b200.query_strategies.strategy import Strategy
    assert "MarginClusteringSampler" in ACCELERATED and "MarginClusteringSampler" not in NOT_ON_THIS_PATH
    assert get_strategy("MarginClusteringSampler").__name__ == "MarginClusteringSampler"
    assert "MarginClusteringSampler" in make_drop_in(Strategy)
