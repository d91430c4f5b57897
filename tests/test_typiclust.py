"""TypiClustSampler without a GPU: the oracle's selection against the authors' loop, its seeding against al_oracle's D^2
cold start, its k-means fixed point, K15's band against fp64 truth, and the sampler's host logic (RNG draws, budget
clamp, K, dropped and exhausted clusters, a gloo world of 2) through a fake engine built on the oracle."""
import os

import numpy as np
import pytest
import torch

import probcover_oracle as P
import typiclust_oracle as T
from helpers import OracleEngine, make_strategy
from oracle import al_oracle as O


def _exact_rows(rng, n, d, nnz=4):
    """Rows with `nnz` entries of +-1: normalised, every entry is +-1/sqrt(nnz) exactly (nnz a square), so every fp32
    dot product and norm is exact in any order."""
    x = np.zeros((n, d), dtype=np.float32)
    for i in range(n):
        x[i, rng.choice(d, nnz, replace=False)] = rng.choice([-1.0, 1.0], nnz)
    return x


def test_oracle_selection_equals_the_authors_loop_while_no_cluster_runs_dry():
    rng = np.random.default_rng(0)
    checked = 0
    for trial in range(60):
        n = int(rng.integers(20, 160))
        d = int(rng.integers(2, 6))
        k = int(rng.integers(1, 12))
        nl = int(rng.integers(0, n // 3))
        feats = rng.normal(size=(n, d)).astype(np.float32)
        if trial % 3 == 1:
            feats[rng.integers(0, n, n // 4)] = feats[0]              # duplicate rows: zero distances, typicality ties
        labels = rng.integers(0, k, n)
        is_lab = np.arange(n) < nl                                    # the authors' labeled rows come first
        avail = ~is_lab
        order = T.cluster_order(labels, is_lab, k)
        if not len(order):
            continue
        room = min(int((avail & (labels == c)).sum()) for c in order)
        if room == 0:
            continue
        budget = int(rng.integers(1, room * len(order) + 1))
        mine = T.select(feats, labels, k, is_lab, avail, budget)
        theirs = T.authors_select(feats, labels, nl, budget)
        assert mine.tolist() == theirs.tolist()
        checked += 1
    assert checked >= 30


def test_seeding_equals_the_d2_cold_start_of_al_oracle():
    rng = np.random.default_rng(1)
    for n, d, k in ((50, 8, 7), (200, 16, 40), (64, 36, 64)):
        xhat = T.normalize(_exact_rows(rng, n, d))
        np.random.seed(n + k)
        first = int(np.random.choice(n))
        got = T.seed(xhat, first, np.random.random_sample(k - 1), k)
        after = np.random.get_state()
        np.random.seed(n + k)
        want = O.coreset(O.pairwise_l2_dist(torch.from_numpy(xhat)), np.zeros(n, dtype=bool), k, randomize=True)
        assert got.tolist() == want
        assert (np.random.get_state()[1] == after[1]).all() and np.random.get_state()[2] == after[2]
        assert len(set(got.tolist())) == k


def test_kmeans_ends_at_a_fixed_point():
    rng = np.random.default_rng(2)
    for n, d, k in ((300, 8, 12), (500, 28, 40), (120, 4, 1)):
        c = rng.normal(size=(max(k // 2, 1), d))
        x = (c[rng.integers(0, len(c), n)] + 0.3 * rng.normal(size=(n, d))).astype(np.float32)
        xhat = T.normalize(x)
        labels, centres, it = T.kmeans(xhat, int(rng.integers(n)), rng.random(k - 1), k)
        assert it < T.MAX_ITER
        assert (T.assign(xhat, centres) == labels).all()
        for cl in np.unique(labels):
            rows = np.flatnonzero(labels == cl)
            s = np.zeros(d)
            for r in rows:
                s = s + xhat[r].astype(np.float64)
            assert (centres[cl] == (s / len(rows)).astype(np.float32)).all()
    assert T.lloyd(xhat, xhat[:1].copy(), max_iter=1)[2] == 1


@pytest.mark.parametrize("d", [4, 28, 64, 520, 2048])
def test_assign_band_holds_for_centres_inside_the_unit_ball(d):
    """The rows of the bound families against centres that are means of them (norm < 1), under the three adder models:
    |g - fsum| <= E with the centre's own norm, and every row the band decides gets the exact argmin."""
    rng = np.random.default_rng(200 + d)
    fam = P.bound_families(rng, d, instances=2)
    xh = np.concatenate(list(fam.values()))
    picks = [rng.choice(len(xh), int(rng.integers(2, 9)), replace=False) for _ in range(24)]
    cen = np.stack([xh[p].astype(np.float64).mean(axis=0) for p in picks]).astype(np.float32)
    cen = np.concatenate([cen, 0.5 * xh[:4], xh[5:6]])                 # a centre on a row: d2 = 0
    cn = P.nrm2(cen)
    assert (cn[:24] < 1.0).all()
    i, j = np.meshgrid(np.arange(len(xh)), np.arange(len(cen)), indexing="ij")
    i, j = i.ravel(), j.ravel()
    truth = P.exact_dots(xh[i], cen[j])
    nx = P.nrm2(xh)
    bound = P.screen_bound(d, nx[i], cn[j])
    want = T.assign(xh, cen)
    for adder in ("nearest", "zero", "align"):
        g = P.emulate_3xtf32(xh[i], cen[j], adder=adder)
        assert (np.abs(g.astype(np.float64) - truth) <= bound).all(), adder
        ok, c1 = T.assign_decide(d, nx, cn, g.reshape(len(xh), len(cen)))
        assert (c1[ok] == want[ok]).all() and ok.any()


# ---- the sampler's host logic ------------------------------------------------------------------------------------------
class TypiClustEngine(OracleEngine):
    """The oracle engine plus normalize / kmeans / typicality by the NumPy statement; records each K."""

    def __init__(self):
        self.ks = []
        self.typicality_calls = 0

    def normalize(self, x):
        return torch.from_numpy(T.normalize(x.numpy()))

    def kmeans(self, xhat, first_pick, uniforms, k, max_iter=T.MAX_ITER):
        self.ks.append(int(k))
        x = xhat.numpy()
        seeds = T.seed(x, first_pick, uniforms, k)
        labels, centres, it = T.lloyd(x, x[seeds].copy(), max_iter)
        return torch.from_numpy(labels.astype(np.int32)), torch.from_numpy(centres), it, seeds

    def typicality(self, xhat, rows, group_off, k=20):
        self.typicality_calls += 1
        rows = rows.numpy()
        typ, best = [], []
        for g in range(len(group_off) - 1):
            t = T.typicality(xhat.numpy(), rows[group_off[g]:group_off[g + 1]], k)
            typ.append(t)
            best.append(int(group_off[g]) + int(np.argmax(t)))
        return torch.from_numpy(np.concatenate(typ)), np.asarray(best, dtype=np.int64)


def _pool(n=160, d=6, seed=3, n_lab=9):
    rng = np.random.default_rng(seed)
    c = rng.normal(size=(12, d))
    emb = torch.from_numpy((c[rng.integers(0, 12, n)] + 0.4 * rng.normal(size=(n, d))).astype(np.float32))
    logits = torch.zeros(n, 4)
    eval_idxs = rng.choice(n, 12, replace=False)
    rest = np.setdiff1d(np.arange(n), eval_idxs)
    labeled = rng.choice(rest, n_lab, replace=False)
    return emb, logits, eval_idxs, labeled


def _expected(s, emb, budget):
    """What the query returns, replayed from the same RNG state: the two shuffles, then the oracle."""
    union = np.asarray(s.get_idxs_for_coreset(), dtype=np.int64)
    is_lab = s.already_labeled_idxs(boolean=True)[union]
    avail = s.available_query_idxs(boolean=True)[union]
    return union[T.query_positions(emb.numpy()[union], is_lab, avail, budget)].tolist()


@pytest.mark.parametrize("budget", [1, 7, 25, 60, 10 ** 6])
def test_query_equals_the_oracle_with_numpys_draws(budget):
    emb, logits, ev, lab = _pool()
    eng = TypiClustEngine()
    s = make_strategy("TypiClustSampler", logits, emb, ev, lab, 32, engine=eng)
    np.random.seed(11)
    got, k = s.query(budget)
    state = np.random.get_state()
    np.random.seed(11)
    want = _expected(s, emb, budget)
    assert got == want and k == len(want)
    assert k == min(budget, int(s.available_query_idxs(boolean=True).sum()))
    assert len(set(got)) == k and not s.idxs_lb[got].any() and not np.isin(got, ev).any()
    after = np.random.get_state()
    assert state[2] == after[2] and (state[1] == after[1]).all()
    assert eng.ks == [min(len(lab) + k, T.MAX_NUM_CLUSTERS)]


def test_zero_budget_returns_nothing_and_draws_only_the_pool():
    emb, logits, ev, lab = _pool()
    eng = TypiClustEngine()
    s = make_strategy("TypiClustSampler", logits, emb, ev, lab, 32, engine=eng)
    for budget in (0, -3):
        np.random.seed(5)
        assert s.query(budget) == ([], 0)
        state = np.random.get_state()
        np.random.seed(5)
        s.get_idxs_for_coreset()
        assert (np.random.get_state()[1] == state[1]).all() and np.random.get_state()[2] == state[2]
    assert eng.ks == []


def test_k_at_and_above_the_cluster_cap(monkeypatch):
    emb, logits, ev, lab = _pool(n=400, n_lab=30)
    for cap, budget in ((40, 10), (40, 11), (40, 50)):
        monkeypatch.setattr(T, "MAX_NUM_CLUSTERS", cap)
        eng = TypiClustEngine()
        s = make_strategy("TypiClustSampler", logits, emb, ev, lab, 32, engine=eng)
        s.MAX_NUM_CLUSTERS = cap
        np.random.seed(3)
        got, _ = s.query(budget)
        np.random.seed(3)
        assert got == _expected(s, emb, budget)
        assert eng.ks == [min(30 + budget, cap)]


def _walk_case(seed, n, sizes, budget, n_lab=0):
    """A query whose clusters are given: labels by `sizes`, rows spread so the k-means of the fake engine returns them."""
    rng = np.random.default_rng(seed)
    k = len(sizes)
    labels = np.repeat(np.arange(k), sizes)
    rng.shuffle(labels)
    xhat = T.normalize(rng.normal(size=(n, 5)).astype(np.float32))
    is_lab = np.zeros(n, dtype=bool)
    is_lab[rng.choice(n, n_lab, replace=False)] = True
    return xhat, labels, k, is_lab, ~is_lab, budget


def test_small_clusters_are_dropped_and_exhausted_ones_skipped():
    xhat, labels, k, is_lab, avail, _ = _walk_case(4, 60, [5, 20, 8, 6, 1, 20], 0, n_lab=6)
    order = T.cluster_order(labels, is_lab, k)
    assert 0 not in order and 4 not in order and sorted(order.tolist()) == [1, 2, 3, 5]
    picks = T.select(xhat, labels, k, is_lab, avail, 10 ** 6)
    kept = np.isin(labels, order)
    assert sorted(picks.tolist()) == np.flatnonzero(kept & avail).tolist()    # every kept row, then nothing
    assert not np.isin(labels[picks], [0, 4]).any()
    # the walk of the sampler (one typicality launch per cycle) visits in the same order
    eng = TypiClustEngine()
    s = make_strategy("TypiClustSampler", torch.zeros(60, 4), torch.zeros(60, 5), [], [], 32, engine=eng)
    for budget in (1, 4, 9, 37, 10 ** 6):
        want = T.select(xhat, labels, k, is_lab, avail, budget)
        eng.typicality_calls = 0
        got = s._walk(torch.from_numpy(xhat), labels, is_lab, avail, budget)
        assert got.tolist() == want.tolist()
        assert eng.typicality_calls == np.bincount(labels[want]).max()          # one launch per cycle


def test_exhausted_clusters_fill_at_random():
    emb, logits, ev, lab = _pool(n=90, n_lab=4)
    eng = TypiClustEngine()
    s = make_strategy("TypiClustSampler", logits, emb, ev, lab, 32, engine=eng)
    np.random.seed(21)
    got, k = s.query(70)
    state = np.random.get_state()
    np.random.seed(21)
    assert got == _expected(s, emb, 70) and k == 70 and len(set(got)) == 70
    assert (np.random.get_state()[1] == state[1]).all() and np.random.get_state()[2] == state[2]


def _one_query():
    emb, logits, ev, lab = _pool()
    return make_strategy("TypiClustSampler", logits, emb, ev, lab, 32, engine=TypiClustEngine())


def _worker(rank, world, port, out_path):
    import os
    import sys
    import torch.distributed as dist
    here = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, os.path.dirname(here))
    sys.path.insert(0, here)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from active_learning_b200.sharding import ShardGroup
    from test_typiclust import _one_query
    s = _one_query()
    s._shard_group = ShardGroup()
    np.random.seed(9)
    res = s.query(40)
    all_res = [None] * world
    dist.all_gather_object(all_res, res)
    if rank == 0:
        np.save(out_path, np.array(all_res, dtype=object), allow_pickle=True)
    dist.barrier()
    dist.destroy_process_group()


def test_world_size_two_returns_the_one_rank_picks_on_every_rank():
    import socket
    import tempfile
    import torch.multiprocessing as mp
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    out = os.path.join(tempfile.mkdtemp(), "res.npy")
    mp.spawn(_worker, args=(2, port, out), nprocs=2, join=True)
    np.random.seed(9)
    want = _one_query().query(40)
    for got in np.load(out, allow_pickle=True):
        assert tuple(got) == tuple(want)
