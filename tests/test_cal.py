"""CALSampler without a GPU: the oracle's picks against the authors' loop, its k-NN against brute force, K18's band against
fp64 truth for unnormalised rows, and the sampler's host logic (RNG draws, budget clamp, k > M, M = 0, the embedding cache,
a gloo world of 2) through a fake engine built on the oracle."""
import os

import numpy as np
import pytest
import torch

import cal_oracle as CO
import probcover_oracle as P
from helpers import FakeExperiment, IndexDataset, OracleEngine, make_strategy


def _authors_fixture(seed, n_lab, n_cand, d, c, budget, k):
    """Embeddings and logits whose k-th / (k + 1)-th neighbour distances and whose scores at the cut are well separated,
    or None."""
    rng = np.random.default_rng(seed)
    emb = rng.normal(size=(n_lab + n_cand, d)).astype(np.float32)
    logits = (rng.normal(size=(n_lab + n_cand, c)) * 2.0).astype(np.float32)
    lab, cand = np.arange(n_lab), np.arange(n_lab, n_lab + n_cand)
    full = np.stack([CO.exact_d2(np.repeat(emb[i:i + 1], n_lab, axis=0), emb[lab]) for i in cand])
    srt = np.sort(full, axis=1)
    if (srt[:, k] - srt[:, k - 1] <= 1e-3 * srt[:, k]).any():
        return None
    idx, _ = CO.knn(emb[cand], emb[lab], k)
    sc = np.sort(CO.scores(logits[cand], logits[lab], idx))[::-1]
    if sc[budget - 1] - sc[budget] <= 1e-4 * abs(sc[budget - 1]):
        return None
    return emb, logits, lab, cand


def test_oracle_picks_equal_the_authors_loop_on_separated_fixtures():
    checked = 0
    for seed in range(80):
        rng = np.random.default_rng(1000 + seed)
        n_lab, n_cand = int(rng.integers(12, 60)), int(rng.integers(30, 120))
        d, c = int(rng.integers(2, 9)), int(rng.choice([2, 3, 10]))
        k = min(CO.NUM_NEIGHBORS, n_lab)
        budget = int(rng.integers(1, n_cand))
        fx = _authors_fixture(seed, n_lab, n_cand, d, c, budget, k)
        if fx is None:
            continue
        emb, logits, lab, cand = fx
        is_lab = np.zeros(len(emb), dtype=bool)
        is_lab[lab] = True
        mine = CO.query_positions(emb, logits, is_lab, ~is_lab, budget)
        theirs = CO.authors_select(emb[lab], logits[lab], emb[cand], logits[cand], budget, k)
        assert sorted(mine.tolist()) == sorted(cand[theirs].tolist())
        checked += 1
    assert checked >= 20


@pytest.mark.parametrize("k", [1, 3, 10, 32])
def test_oracle_knn_equals_brute_force(k):
    rng = np.random.default_rng(k)
    for n, m, d in ((40, 50, 4), (33, 7, 12), (25, 120, 28)):
        x = rng.integers(-3, 4, size=(n, d)).astype(np.float32)          # small integers: exact ties everywhere
        y = rng.integers(-3, 4, size=(m, d)).astype(np.float32)
        y[m // 2:m // 2 + 3] = y[1]                                      # duplicated references, before and after
        x[0] = y[m - 1]                                                  # d2 = 0
        x[1] = (rng.normal(size=d) * 1e3).astype(np.float32)             # mixed norms
        idx, d2 = CO.knn(x, y, k)
        for i in range(n):
            e = CO.exact_d2(np.repeat(x[i:i + 1], m, axis=0), y)
            o = np.lexsort((np.arange(m), e))[:k]
            kk = min(k, m)
            assert idx[i, :kk].tolist() == o.tolist() and d2[i, :kk].tolist() == e[o].tolist()
            assert (idx[i, kk:] == -1).all() and np.isinf(d2[i, kk:]).all()      # k > M
        assert d2[0, 0] == 0.0


@pytest.mark.parametrize("d", [4, 28, 64, 520, 2048])
def test_band_holds_for_unnormalised_rows(d):
    """The bound families rescaled to norms between 1e-3 and 1e3, under the three adder models: |g - <x, y>| <= E, and the
    screen's d2~ lies within K18's band of the exact value."""
    rng = np.random.default_rng(300 + d)
    xh = np.concatenate(list(P.bound_families(rng, d, instances=2).values()))
    x = (xh * (10.0 ** rng.uniform(-3, 3, size=(len(xh), 1)))).astype(np.float32)
    y = (xh[rng.permutation(len(xh))] * (10.0 ** rng.uniform(-3, 3, size=(len(xh), 1)))).astype(np.float32)
    y[:3] = x[:3]                                                        # exact duplicates: d2 = 0
    i, j = np.meshgrid(np.arange(len(x)), np.arange(len(y)), indexing="ij")
    i, j = i.ravel(), j.ravel()
    nx, ny = P.nrm2(x), P.nrm2(y)
    truth = P.exact_dots(x[i], y[j])
    e = CO.exact_d2(x[i], y[j])
    b = CO.band(d, nx[i], ny[j])
    for adder in ("nearest", "zero", "align"):
        g = P.emulate_3xtf32(x[i], y[j], adder=adder)
        assert (np.abs(g.astype(np.float64) - truth) <= P.screen_bound(d, nx[i], ny[j])).all(), adder
        assert (np.abs(CO.screen_d2(nx[i], ny[j], g) - e) <= b).all(), adder


def test_score_keys_and_order():
    """A zero score's key is +0.0, so zero scores tie by position; NaN sorts last; larger scores come first."""
    s = np.array([0.0, 1.5, 0.0, np.nan, 1.5, 2.0, -0.0])
    key = CO.keys(s)
    assert not np.signbit(key[[0, 2, 6]]).any()
    assert CO.select(key, 7).tolist() == [5, 1, 4, 0, 2, 6, 3]


# ---- the sampler's host logic ------------------------------------------------------------------------------------------
class CALEngine(OracleEngine):
    """The oracle engine plus knn / cal_scores by the NumPy statement; records each k."""

    def __init__(self):
        self.ks = []

    def knn(self, x, y, k):
        self.ks.append(int(k))
        idx, d2 = CO.knn(x.numpy(), y.numpy(), int(k))
        return torch.from_numpy(idx.astype(np.int32)), torch.from_numpy(d2), 0

    def cal_scores(self, cand_logits, ref_logits, idx):
        s = CO.scores(cand_logits.numpy(), ref_logits.numpy(), idx.numpy())
        return torch.from_numpy(s), torch.from_numpy(CO.keys(s))


def _pool(n=160, d=6, c=5, seed=3, n_lab=20):
    rng = np.random.default_rng(seed)
    emb = torch.from_numpy(rng.normal(size=(n, d)).astype(np.float32))
    logits = torch.from_numpy((rng.normal(size=(n, c)) * 2).astype(np.float32))
    eval_idxs = rng.choice(n, 12, replace=False)
    rest = np.setdiff1d(np.arange(n), eval_idxs)
    labeled = rng.choice(rest, n_lab, replace=False)
    return emb, logits, eval_idxs, labeled


def _expected(s, emb, logits, budget):
    """What the query returns, replayed from the same RNG state: the two shuffles, then the oracle."""
    union = np.asarray(s.get_idxs_for_coreset(), dtype=np.int64)
    is_lab = s.already_labeled_idxs(boolean=True)[union]
    avail = s.available_query_idxs(boolean=True)[union]
    return union[CO.query_positions(emb.numpy()[union], logits.numpy()[union], is_lab, avail, budget)].tolist()


@pytest.mark.parametrize("n_lab,budget", [(20, 1), (20, 17), (20, 10 ** 6), (4, 30), (2, 5)])
def test_query_equals_the_oracle_and_draws_only_the_shuffles(n_lab, budget):
    emb, logits, ev, lab = _pool(n_lab=n_lab)
    eng = CALEngine()
    s = make_strategy("CALSampler", logits, emb, ev, lab, 32, engine=eng)
    np.random.seed(11)
    got, k = s.query(budget)
    state = np.random.get_state()
    np.random.seed(11)
    want = _expected(s, emb, logits, budget)
    assert got == want and k == len(want)
    assert k == min(budget, int(s.available_query_idxs(boolean=True).sum()))
    assert len(set(got)) == k and not s.idxs_lb[got].any() and not np.isin(got, ev).any()
    np.random.seed(11)
    s.get_idxs_for_coreset()
    after = np.random.get_state()
    assert state[2] == after[2] and (state[1] == after[1]).all()
    assert eng.ks == [min(n_lab, CO.NUM_NEIGHBORS)]                       # k = min(10, M): k > M gives k = M


def test_zero_budget_and_no_labeled_rows():
    emb, logits, ev, lab = _pool()
    for labeled in (lab, []):
        eng = CALEngine()
        s = make_strategy("CALSampler", logits, emb, ev, labeled, 32, engine=eng)
        for budget in (0, -3):
            np.random.seed(5)
            assert s.query(budget) == ([], 0)
            state = np.random.get_state()
            np.random.seed(5)
            s.get_idxs_for_coreset()
            assert (np.random.get_state()[1] == state[1]).all() and np.random.get_state()[2] == state[2]
        assert eng.ks == []
    with pytest.raises(ValueError, match="CALSampler"):
        s.query(10)


class _Enc(torch.nn.Module):
    """The pool index -> its embedding (a buffer, so the cache's fingerprint sees it)."""

    def __init__(self, emb):
        super().__init__()
        self.register_buffer("table", emb.clone())

    def forward(self, x):
        return self.table[x.long()]


class _EncoderNet(torch.nn.Module):
    """resnet_simclr.py's layout with integer embeddings and head: every logit is exact in any order."""

    def __init__(self, emb, c, seed):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.encoder = _Enc(emb)
        self.linear = torch.nn.Linear(emb.shape[1], c)
        with torch.no_grad():
            self.linear.weight.copy_(torch.randint(-2, 3, (c, emb.shape[1]), generator=g).float())
            self.linear.bias.copy_(torch.randint(-2, 3, (c,), generator=g).float())
        self.encoder_rows = 0

    def forward(self, x, return_features=False, specify_input_layer=None):
        h = self.encoder(x)
        self.encoder_rows += len(x)
        out = self.linear(h)
        return (out, h) if return_features else out


@pytest.mark.parametrize("cache", [True, False])
def test_query_over_two_rounds_with_and_without_the_embedding_cache(cache):
    n, c = 300, 7
    rng = np.random.default_rng(8)
    emb = torch.from_numpy(rng.integers(-4, 5, size=(n, 6)).astype(np.float32))
    net = _EncoderNet(emb, c, 8)
    ev = rng.choice(n, 20, replace=False)
    lab = rng.choice(np.setdiff1d(np.arange(n), ev), 25, replace=False)
    s = make_strategy("CALSampler", torch.zeros(n, c), emb, ev, lab, 32, engine=CALEngine(), net=None,
                      freeze_feature=cache, cache_embeddings=cache)
    s.net = s.feature_net = net
    for rnd, budget in enumerate((15, 40)):
        with torch.no_grad():
            logits = net.linear(emb)
        np.random.seed(40 + rnd)
        got, k = s.query(budget)
        np.random.seed(40 + rnd)
        assert got == _expected(s, emb, logits, budget) and k == budget
        s.update(got, k)
        with torch.no_grad():                                            # "training" moves the head only
            net.linear.bias.add_(1.0)
    assert (getattr(s, "_emb_cache", None) is not None) == cache
    assert (net.encoder_rows == 0) == cache                              # cached: the encoder alone, once per row


def _one_query():
    emb, logits, ev, lab = _pool()
    return make_strategy("CALSampler", logits, emb, ev, lab, 32, engine=CALEngine())


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
    from test_cal import _one_query
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
