"""Host logic of the drop-in samplers on CPU (OracleEngine injected): index bookkeeping, RNG
consumption order, partition batching, dispatch, pickling.  Reference outputs come from
tests/golden/reference_golden.npz."""
import pickle

import numpy as np
import pytest
import torch

from helpers import OracleEngine, make_strategy
from oracle import al_oracle as O


def _pool(gold):
    return int(gold["e2e_n"]), gold["e2e_eval_idxs"], gold["e2e_labeled"]


def test_dispatch_names_match_reference():
    from active_learning_b200.query_strategies.get_strategy import (ACCELERATED, NOT_ON_THIS_PATH,
                                                                    get_strategy)
    for name in ACCELERATED + ("RandomSampler",):
        assert get_strategy(name).__name__ == name
    for name in NOT_ON_THIS_PATH:
        with pytest.raises(NotImplementedError):
            get_strategy(name)(None)
    with pytest.raises(NameError):
        get_strategy("NoSuchSampler")


def test_no_engine_without_gpu_is_loud(gold):
    """Product path: no CUDA device -> the sampler raises, it never falls back to CPU."""
    if torch.cuda.is_available():
        pytest.skip("needs a CPU-only box")
    n, ev, lab = _pool(gold)
    s = make_strategy("MarginSampler", torch.from_numpy(gold["margin_f32_c10_logits"]),
                      torch.zeros(n, 4), ev, lab, 128)
    from active_learning_b200._lib import AlqError
    with pytest.raises(AlqError):
        s.query(10.0)


def test_margin_and_confidence_plumbing(gold):
    n, ev, lab = _pool(gold)
    for tag in ("f32_c10", "f32_c1000"):
        s = make_strategy("MarginSampler", torch.from_numpy(gold[f"margin_{tag}_logits"]),
                          torch.zeros(n, 4), ev, lab, 128, engine=OracleEngine())
        np.random.seed(7)
        idx, cost = s.query(60.0)                      # budget arrives as a float (parser.py:46)
        assert idx == gold[f"margin_{tag}_picks"].tolist() and cost == 60
        assert all(isinstance(i, int) for i in idx)
        assert s.net.training                          # margin_sampler.py:38
    s = make_strategy("ConfidenceSampler", torch.from_numpy(gold["confidence_f32_logits"]),
                      torch.zeros(n, 4), ev, lab, 128, engine=OracleEngine())
    np.random.seed(7)
    idx, _ = s.query(60.0)
    assert idx == gold["confidence_f32_picks"].tolist()
    s.update(idx, len(idx))                            # strategy.py:470 assertion holds


def test_entropy_sampler_config0_plumbing():
    """BASELINE config 0: EntropySampler, CIFAR-shaped pool of 1k, budget 100, one round (CPU)."""
    torch.manual_seed(0)
    n = 1000
    logits = torch.randn(n, 10) * 2
    s = make_strategy("EntropySampler", logits, torch.zeros(n, 4), np.arange(10), [], 100,
                      engine=OracleEngine())
    idx, cost = s.query(100.0)
    assert cost == 100 and len(set(idx)) == 100 and not set(idx) & set(range(10))
    ent = -(torch.softmax(logits, 1) * torch.log_softmax(logits, 1)).sum(1)
    pool = np.arange(10, n)
    top = pool[np.argsort(-ent[pool].numpy(), kind="stable")[:100]]
    assert set(idx) == set(top.tolist())
    s.update(idx, cost)
    assert s.idxs_lb.sum() == 100


@pytest.mark.parametrize("name,sub,parts", [("CoresetSampler", False, 1), ("CoresetSampler", True, 1),
                                            ("PartitionedCoresetSampler", True, 3),
                                            ("BADGESampler", True, 1),
                                            ("PartitionedBADGESampler", True, 3)])
@pytest.mark.parametrize("etag", ["int", "f32"])
def test_coreset_family_plumbing(gold, name, sub, parts, etag):
    n, ev, lab = _pool(gold)
    kw = dict(partitions=parts)
    if sub:
        kw.update(subset_labeled=60, subset_unlabeled=300)
    s = make_strategy(name, torch.from_numpy(gold["e2e_logits"]),
                      torch.from_numpy(gold[f"e2e_emb_{etag}"]), ev, lab, 64, engine=OracleEngine(), **kw)
    np.random.seed(21)
    idx, cost = s.query(50.0)
    ref = gold[f"e2e_{name}_{'sub' if sub else 'all'}_{etag}"].tolist()
    assert cost == 50
    assert [int(i) for i in idx] == ref
    s.update(idx, cost)


def test_cold_start_partitions_consume_rng_like_reference(gold):
    """Nothing labeled: first centre by np.random.choice(n) (BADGE) / minimax (CoreSet); the
    oracle's dense `coreset` on the same rows is the reference behaviour (pinned in
    test_oracle_golden)."""
    n, ev, _ = _pool(gold)
    emb = torch.from_numpy(gold["e2e_emb_int"])
    logits = torch.from_numpy(gold["e2e_logits"])
    for name, rand in (("CoresetSampler", False), ("BADGESampler", True)):
        s = make_strategy(name, logits, emb, ev, [], 64, engine=OracleEngine())
        np.random.seed(5)
        idx, _ = s.query(12.0)
        np.random.seed(5)
        union, _, _ = O.idxs_for_coreset(np.zeros(n, dtype=bool), ev, None, None)
        feats = emb[union] if not rand else O.gradient_embeddings(logits[union], emb[union], 64)
        ref = O.coreset(O.pairwise_l2_dist(feats), np.zeros(len(union), dtype=bool), 12, randomize=rand)
        assert idx == np.array(union)[ref].tolist()


def test_strategy_pickles_without_engine(gold):
    n, ev, lab = _pool(gold)
    s = make_strategy("CoresetSampler", torch.from_numpy(gold["e2e_logits"]),
                      torch.from_numpy(gold["e2e_emb_int"]), ev, lab, 64, engine=OracleEngine())
    np.random.seed(1)
    s.query(5.0)
    assert s._saved_embeddings is not None            # freeze_feature cache (coreset_sampler.py:120)
    blob = pickle.dumps(s)                             # utils/resume_training.py:49
    t = pickle.loads(blob)
    assert t._engine is None and getattr(t, "_saved_embeddings", None) is None
    assert (t.idxs_lb == s.idxs_lb).all()


def test_update_refuses_relabel(gold):
    n, ev, lab = _pool(gold)
    s = make_strategy("RandomSampler", torch.zeros(n, 10), torch.zeros(n, 4), ev, lab, 64)
    with pytest.raises(AssertionError):
        s.update([int(lab[0])], 1)
    np.random.seed(3)
    idx, cost = s.query(25)
    assert cost == 25 and not set(idx) & set(lab.tolist()) and not set(idx) & set(ev.tolist())


def test_drop_in_binding_on_foreign_base(gold):
    """make_drop_in puts the accelerated query() on any Strategy-shaped base class."""
    from active_learning_b200.integration import make_drop_in
    from active_learning_b200.query_strategies.strategy import Strategy

    class ForeignStrategy(Strategy):
        marker = "reference-base"

    cls = make_drop_in(ForeignStrategy)
    assert set(cls) >= {"MarginSampler", "CoresetSampler", "BADGESampler"}
    assert ForeignStrategy in cls["MarginSampler"].__mro__
    assert cls["MarginSampler"].query is not ForeignStrategy.query


class _EncoderNet(torch.nn.Module):
    """resnet_simclr.py layout: encoder -> (detached) -> linear; the forward counts encoder calls."""

    def __init__(self, n_pool, d, c):
        super().__init__()
        self.table = torch.nn.Embedding(n_pool, d)
        self.encoder = torch.nn.Sequential(torch.nn.Linear(d, d), torch.nn.ReLU())
        self.linear = torch.nn.Linear(d, c)
        self.encoder_rows = 0

    def forward(self, x, return_features=False, specify_input_layer=None):
        self.encoder_rows += len(x)
        h = self.encoder(self.table(x.long())).detach()
        out = self.linear(h)
        return (out, h) if return_features else out


def test_embedding_cache_across_rounds_matches_uncached():
    """--freeze_feature: the encoder runs once per pool row over all rounds; picks equal the uncached run
    even after the linear head changes between rounds (section 8f rank 1)."""
    from helpers import FakeExperiment, IndexDataset
    from active_learning_b200.query_strategies.get_strategy import get_strategy
    import tempfile
    n, d, c = 400, 16, 10
    results = {}
    for cached in (False, True):
        torch.manual_seed(0)
        net = _EncoderNet(n, d, c)

        class CountingEncoder(torch.nn.Module):
            def __init__(self, inner):
                super().__init__()
                self.inner, self.rows = inner, 0

            def forward(self, x):
                self.rows += len(x)
                return self.inner(x)

        ds = IndexDataset(n, c)
        orig_getitem = ds.__getitem__

        class DS(IndexDataset):
            def __getitem__(self, i):
                return net.table.weight.detach()[i].clone(), 0, i
        ds = DS(n, c)
        net.encoder = CountingEncoder(net.encoder)

        class Net2(torch.nn.Module):
            def __init__(self, enc, lin):
                super().__init__()
                self.encoder, self.linear = enc, lin

            def forward(self, x, return_features=False, specify_input_layer=None):
                h = self.encoder(x).detach()
                o = self.linear(h)
                return (o, h) if return_features else o
        net2 = Net2(net.encoder, net.linear)
        picks = []
        for name in ("MarginSampler", "CoresetSampler", "BADGESampler"):
            args = dict(early_stop_patience=0, n_epoch=1, world_size=1, model="m", freeze_feature=True,
                        ckpt_path=tempfile.mkdtemp(), exp_name="t", subset_labeled=None, subset_unlabeled=None,
                        partitions=1, cache_embeddings=cached)
            s = get_strategy(name)(ds, ds, net2, {"loader_te_args": {"batch_size": 32, "num_workers": 0}},
                                   np.arange(5), FakeExperiment(), None, **args)
            s.init_network_weights()
            s.set_engine(OracleEngine())
            s.update(np.arange(5, 45), 40)
            net2.encoder.rows = 0
            for rd in range(3):
                np.random.seed(rd)
                idx, cost = s.query(20.0)
                s.update(idx, cost)
                picks.append(idx)
                with torch.no_grad():                       # "training" moves only the head
                    net2.linear.weight.add_(0.01 * (rd + 1))
            if cached:
                assert net2.encoder.rows <= n, (name, net2.encoder.rows)   # each pool row encoded at most once
            elif name != "CoresetSampler":    # (CoreSet keeps the reference's own per-strategy cache, coreset_sampler.py:120)
                assert net2.encoder.rows > n
        results[cached] = picks
    assert results[True] == results[False]


# ---- MASE / BASE (SURVEY.md section 8f rank 2) -------------------------------------------------------
@pytest.fixture(scope="module")
def mgold():
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    return dict(np.load(os.path.join(root, "tests", "golden", "reference_golden_mase.npz")))


def _mase_strategy(name, g, tag, engine):
    from helpers import HeadNet
    net = HeadNet(torch.from_numpy(g[f"{tag}_emb"]), torch.from_numpy(g[f"{tag}_weight"]),
                  torch.from_numpy(g[f"{tag}_bias"]))
    return make_strategy(name, None, None, g[f"{tag}_eval"], g[f"{tag}_labeled"], int(g[f"{tag}_bs"]),
                         engine=engine, net=net)


@pytest.mark.parametrize("tag", ["a", "b"])
def test_mase_base_plumbing(mgold, tag):
    g = mgold
    budget = float(g[f"{tag}_budget"])
    for name, key in (("MASESampler", "mase_picks"), ("BASESampler", "base_picks")):
        s = _mase_strategy(name, g, tag, OracleEngine())
        st0 = np.random.get_state()[1].copy()
        idx, cost = s.query(budget)
        assert idx == g[f"{tag}_{key}"].tolist() and cost == int(budget)
        assert all(isinstance(i, int) for i in idx)
        assert (np.random.get_state()[1] == st0).all()      # shuffle=False: no RNG draw (mase_sampler.py:20)
        s.update(idx, cost)                                 # strategy.py:470 assertion holds
        pickle.dumps(s)
    # compute_margins keeps the reference's 4-tuple API (mase_sampler.py:29,102)
    s = _mase_strategy("MASESampler", g, tag, OracleEngine())
    pool = s.available_query_idxs(boolean=False, shuffle=False)
    mm, pc, pred, true = s.compute_margins(pool)
    assert mm.shape == (len(pool),) and pc.shape == (len(pool), s.num_classes)
    assert pred.dtype == torch.int64 and len(true) == len(pool)
    torch.testing.assert_close(mm, torch.from_numpy(g[f"{tag}_min_margins"]), rtol=1e-4, atol=2e-6)
    # mase_sampler.py:30-33: the augmented train_set can stand in for al_set (same object in this harness)
    mm_aug, _, pred_aug, _ = s.compute_margins(pool, use_training_augmentation=True)
    assert torch.equal(mm_aug, mm) and torch.equal(pred_aug, pred)
    assert s.query(0.0) == ([], 0)


def test_mase_self_check_catches_a_wrong_head(mgold):
    """mase_sampler.py:88-93: if the logits do not come from `linear(finalembed)`, the assertion trips."""
    g = mgold
    s = _mase_strategy("MASESampler", g, "a", OracleEngine())
    real = s.net.forward

    def skewed(x, return_features=False, specify_input_layer=None):
        if specify_input_layer:
            return real(x, specify_input_layer=specify_input_layer) * 1.5 + 0.3 * torch.arange(10.0)
        return real(x, return_features=return_features)
    s.net.forward = skewed
    with pytest.raises(AssertionError):
        s.query(10.0)


def test_update_is_vectorised_with_the_reference_assertion(gold):
    """strategy.py:468-471: labeling an index twice (already labeled, or repeated in the list) asserts."""
    n, ev, lab = _pool(gold)
    s = make_strategy("RandomSampler", torch.zeros(n, 10), torch.zeros(n, 4), ev, lab, 64)
    assert s.idxs_lb.sum() == len(lab) and s.cumulative_cost == len(lab)
    free = np.setdiff1d(np.arange(n), lab)[:5]
    s.update(free.tolist(), 5)                                  # list input (main_al.py:158 passes query()'s list)
    assert s.idxs_lb[free].all() and s.cumulative_cost == len(lab) + 5
    with pytest.raises(AssertionError):
        s.update(np.array([free[0]]), 1)                        # already labeled
    other = np.setdiff1d(np.arange(n), np.flatnonzero(s.idxs_lb))[:2]
    with pytest.raises(AssertionError):
        s.update(np.array([other[0], other[1], other[0]]), 3)   # repeated inside one call
    s.update(np.array([], dtype=np.int64), 0)                   # empty round


class _DecliningTailEngine(OracleEngine):
    """A peer-memory engine whose sharded tail declines the way libalq does when the launch does not fuse and the budget
    exceeds the 16 384 words of the window exchange."""
    comm_ready = True
    declined = 0

    def uncertainty_tail_sharded(self, logits, mode, b, row_lo, rows_min, rows_max, scores_out=None):
        from active_learning_b200._lib import AlqError
        self.declined += 1
        raise AlqError(f"alq_uncertainty_tail_sharded: ALQ_ERR_INVALID: the launch does not fuse and b = {b} exceeds the "
                       f"16384 words of the window exchange")


def test_sharded_uncertainty_query_falls_back_when_the_tail_declines(tmp_path):
    """UncertaintyQuery._query_sharded on a pool whose width never fuses (c = 10) with a budget above 16 384: the sharded
    tail declines, and the query gathers the local winners through ShardGroup.merge_smallest's collective path instead of
    raising.  The picks are the single-process stable selection."""
    import torch.distributed as dist
    from active_learning_b200.sharding import ShardGroup
    n, c, budget = 20000, 10, 17000
    logits = torch.from_numpy(np.random.default_rng(3).integers(-2, 3, size=(n, c)).astype(np.float32))
    eng = _DecliningTailEngine()
    dist.init_process_group("gloo", init_method=f"file://{tmp_path}/init", world_size=1, rank=0)
    try:
        s = make_strategy("MarginSampler", logits, torch.zeros(n, 4), [], [], 4096, engine=eng)
        s._shard_group = ShardGroup()
        idxs = s.available_query_idxs(boolean=False, shuffle=False)
        pos = s._query_sharded(idxs, budget, s._shard_group)
    finally:
        dist.destroy_process_group()
    assert eng.declined == 1
    assert np.array_equal(pos, O.select_smallest(O.softmax_scores(logits, O.MODE_MARGIN, batch_size=4096), budget))
