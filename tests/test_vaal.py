"""VAALSampler without a GPU: the oracle (tests/vaal_oracle.py) against the reference's goldens
(tests/golden/make_golden_vaal.py), and the sampler's host logic -- crop, encoder-only pass, RNG replay, selection order,
module modes, dispatch, pickling, errors, the row-sharded group over gloo -- with a CPU engine that scores with the
discriminator module itself."""
import os
import pickle
import socket
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import vaal_oracle as V
from helpers import HeadNet, OracleEngine, make_strategy

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_vaal as G  # noqa: E402

TAGS = list(G.FIXTURES)


def load_gold():
    return dict(np.load(os.path.join(HERE, "golden", "reference_golden_vaal.npz")))


@pytest.fixture(scope="module")
def vgold():
    return load_gold()


class VAALOracleEngine(OracleEngine):
    """The CPU engine stub with K9 as the discriminator module itself (same layout check as the Engine)."""

    def __init__(self):
        self.p = []

    def vaal_scores(self, mu, discriminator, return_logits=False):
        from active_learning_b200.engine import Engine
        l1 = Engine.vaal_layers(discriminator)[0]
        with torch.no_grad():
            p = discriminator(mu[:, :l1.in_features]).view(-1)
        self.p.append(p)
        return p


def fixture_sampler(gold, tag, engine, **kw):
    """The VAALSampler of golden fixture `tag`, its modules rebuilt from the stored seed, and the fixture's budget."""
    seed = int(gold[f"{tag}_seed"])
    c, _h, _w, _z, n, _ev, _lab, bs, budget = G.FIXTURES[tag]
    ds, ev, lab, crop_seed = G.fixture_inputs(tag, seed)
    vae, disc = G.oracle_modules(tag, seed)
    vae.set_crop_seed(crop_seed)
    net = HeadNet(torch.zeros(n, 4), torch.zeros(c, 4), torch.zeros(c))
    s = make_strategy("VAALSampler", None, None, ev, lab, bs, engine=engine, net=net, dataset=ds, vae=vae,
                      discriminator=disc, **kw)
    return s, budget


def golden_query(gold, s, budget):
    """One query under the golden RNG seeds: (picks, cost, NumPy digest, torch digest)."""
    np.random.seed(int(gold["np_seed"]))
    torch.manual_seed(int(gold["torch_seed"]))
    idx, cost = s.query(float(budget))
    return idx, cost, V.np_rng_digest(), V.torch_rng_digest()


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_replays_the_reference_goldens(vgold, tag):
    s, budget = fixture_sampler(vgold, tag, VAALOracleEngine())
    np.random.seed(int(vgold["np_seed"]))
    torch.manual_seed(int(vgold["torch_seed"]))
    cand = s.available_query_idxs()
    idx, cost, p = V.reference_query(s.al_set, cand, G.FIXTURES[tag][7], s.vae, s.discriminator, float(budget))
    assert idx.tolist() == vgold[f"{tag}_picks"].tolist() and cost == int(vgold[f"{tag}_cost"])
    assert np.array_equal(p, vgold[f"{tag}_p"])
    assert V.np_rng_digest() == str(vgold[f"{tag}_np_digest"])
    assert V.torch_rng_digest() == str(vgold[f"{tag}_torch_digest"])


@pytest.mark.parametrize("tag", TAGS)
def test_sampler_replays_the_reference_goldens(vgold, tag):
    eng = VAALOracleEngine()
    s, budget = fixture_sampler(vgold, tag, eng)
    s.vae.train()
    s.discriminator.train()
    idx, cost, np_d, torch_d = golden_query(vgold, s, budget)
    assert isinstance(idx, np.ndarray) and idx.dtype == np.int64 and isinstance(cost, int)
    assert idx.tolist() == vgold[f"{tag}_picks"].tolist() and cost == int(vgold[f"{tag}_cost"])
    assert np_d == str(vgold[f"{tag}_np_digest"]) and torch_d == str(vgold[f"{tag}_torch_digest"])
    assert not (s.net.training or s.vae.training or s.discriminator.training)
    # the encoder-only pass gives the reference's p (same CPU arithmetic up to the batching of the discriminator)
    np.testing.assert_allclose(eng.p[-1].numpy(), vgold[f"{tag}_p"], rtol=0, atol=1e-6)


def test_crop_window_is_the_reference_rule():
    from active_learning_b200.query_strategies.vaal import crop_window
    for h, w in ((32, 32), (63, 10), (64, 64), (72, 80), (224, 224), (65, 300)):
        for seed in (0, 17, 9999):
            np.random.seed(seed + 1)
            a = crop_window(seed, h, w)
            sa = V.np_rng_digest()
            np.random.seed(seed + 1)
            assert a == V.crop_window(seed, h, w) and sa == V.np_rng_digest()
    for h, w in ((64, 63), (10, 100)):
        with pytest.raises(ValueError):
            crop_window(3, h, w)


def test_budget_zero_and_empty_pool_return_nothing(vgold):
    s, _ = fixture_sampler(vgold, "c", VAALOracleEngine())
    assert s.query(0.0) == ([], 0)
    s.update(s.available_query_idxs(), 0)
    assert s.query(10.0) == ([], 0)


def test_missing_modules_say_how_to_get_them(vgold):
    s, budget = fixture_sampler(vgold, "a", VAALOracleEngine())
    s.discriminator = None
    with pytest.raises(ValueError, match="discriminator="):
        s.query(float(budget))


def test_no_engine_without_gpu_is_loud(vgold):
    if torch.cuda.is_available():
        pytest.skip("needs a CPU-only box")
    from active_learning_b200._lib import AlqError
    s, budget = fixture_sampler(vgold, "a", None)
    with pytest.raises(AlqError):
        s.query(float(budget))


def test_discriminator_layout_is_checked():
    from active_learning_b200._lib import AlqError
    from active_learning_b200.engine import Engine
    good = V.Discriminator(z_dim=7)
    assert [lin.out_features for lin in Engine.vaal_layers(good)] == [512, 512, 1]
    assert len(Engine.vaal_layers(good.net)) == 3
    bad = [torch.nn.Sequential(torch.nn.Linear(7, 256), torch.nn.ReLU(), torch.nn.Linear(256, 512), torch.nn.ReLU(),
                               torch.nn.Linear(512, 1), torch.nn.Sigmoid()),
           torch.nn.Sequential(torch.nn.Linear(7, 512), torch.nn.Tanh(), torch.nn.Linear(512, 512), torch.nn.ReLU(),
                               torch.nn.Linear(512, 1), torch.nn.Sigmoid()),
           torch.nn.Sequential(torch.nn.Linear(7, 512), torch.nn.ReLU(), torch.nn.Linear(512, 512), torch.nn.ReLU(),
                               torch.nn.Linear(512, 1, bias=False), torch.nn.Sigmoid()),
           torch.nn.Linear(7, 1)]
    for m in bad:
        with pytest.raises(AlqError):
            Engine.vaal_layers(m)


def test_pickling_drops_the_engine_and_keeps_the_modules(vgold):
    s, budget = fixture_sampler(vgold, "b", VAALOracleEngine())
    t = pickle.loads(pickle.dumps(s))
    assert t._engine is None and t.vae.crop_seed == s.vae.crop_seed
    t.set_engine(VAALOracleEngine())
    assert golden_query(vgold, t, budget)[0].tolist() == vgold["b_picks"].tolist()


def test_dispatch_and_drop_in_binding(vgold):
    from active_learning_b200.integration import make_drop_in
    from active_learning_b200.query_strategies.get_strategy import ACCELERATED, NOT_ON_THIS_PATH, get_strategy
    from active_learning_b200.query_strategies.strategy import Strategy
    from active_learning_b200.query_strategies.vaal import VAALQuery
    assert "VAALSampler" in ACCELERATED and "VAALSampler" not in NOT_ON_THIS_PATH
    assert get_strategy("VAALSampler").__name__ == "VAALSampler"
    assert "VAALSampler" not in make_drop_in(Strategy)

    seed = int(vgold["a_seed"])

    class RefVAAL(Strategy):
        """Stands in for the reference's VAALSampler: its __init__ builds the modules that its training loop trains."""

        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            self.vae, self.discriminator = G.oracle_modules("a", seed)
            self.vae.set_crop_seed(G.fixture_inputs("a", seed)[3])

        def query(self, budget):
            raise AssertionError("the reference's query must be replaced")

    accel = make_drop_in(Strategy, vaal_base=RefVAAL)
    cls = accel["VAALSampler"]
    assert cls.__bases__ == (VAALQuery, RefVAAL) and set(accel) - {"VAALSampler"} == set(make_drop_in(Strategy))
    c, _h, _w, _z, n, _ev, _lab, bs, budget = G.FIXTURES["a"]
    ds, ev, lab, _ = G.fixture_inputs("a", seed)
    s = cls(ds, ds, HeadNet(torch.zeros(n, 4), torch.zeros(c, 4), torch.zeros(c)),
            {"loader_te_args": {"batch_size": bs, "num_workers": 0}}, ev, None,
            ckpt_path=tempfile.mkdtemp(prefix="alq_test_"))
    s.set_engine(VAALOracleEngine())
    s.update(np.array(lab), len(lab))
    idx, cost, np_d, torch_d = golden_query(vgold, s, budget)
    assert idx.tolist() == vgold["a_picks"].tolist() and torch_d == str(vgold["a_torch_digest"])


def _worker(rank, world, port, out_path):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from active_learning_b200.sharding import ShardGroup
    from test_vaal import VAALOracleEngine, fixture_sampler, golden_query, load_gold
    gold = load_gold()
    group = ShardGroup()
    res = {}
    for tag in TAGS:
        s, budget = fixture_sampler(gold, tag, VAALOracleEngine())
        s._shard_group = group
        idx, cost, np_d, torch_d = golden_query(gold, s, budget)
        res[tag] = (idx.tolist(), cost, np_d, torch_d)
    all_res = [None] * world
    dist.all_gather_object(all_res, res)
    if rank == 0:
        np.save(out_path, np.array(all_res, dtype=object), allow_pickle=True)
    dist.barrier()
    dist.destroy_process_group()


def test_world_size_two_equals_single_process(vgold):
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    out = os.path.join(tempfile.mkdtemp(), "res.npy")
    mp.spawn(_worker, args=(2, port, out), nprocs=2, join=True)
    for res in np.load(out, allow_pickle=True):          # every rank
        for tag in TAGS:
            idx, cost, np_d, torch_d = res[tag]
            assert idx == vgold[f"{tag}_picks"].tolist() and cost == int(vgold[f"{tag}_cost"])
            assert np_d == str(vgold[f"{tag}_np_digest"]) and torch_d == str(vgold[f"{tag}_torch_digest"])
