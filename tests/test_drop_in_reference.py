"""INTEGRATION.md's three-line patch, executed: `make_drop_in` binds the accelerated query() implementations onto a
`Strategy` base class (here the package's own query-path Strategy, which keeps the constructor contract of the
reference's query_strategies/strategy.py:74), the resulting classes are built with that constructor contract and their
query() -- arithmetic by the CPU oracle engine, as everywhere in the CPU tier -- must return exactly what the
reference's own samplers returned on the same pool, labels and RNG seed (tests/golden/make_golden_live.py ran them;
tests/golden/reference_golden_live.npz holds their picks)."""
import os
import sys
import tempfile

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_live as GL        # noqa: E402  (inputs and cases; imports nothing from the reference)


@pytest.fixture(scope="module")
def ref():
    from active_learning_b200.integration import make_drop_in
    from active_learning_b200.query_strategies.strategy import Strategy
    gold = dict(np.load(os.path.join(HERE, "golden", "reference_golden_live.npz")))
    return dict(gold=gold, base=Strategy, accel=make_drop_in(Strategy))


def _build(cls, logits, emb, ev, lab, bs, **kw):
    from helpers import FakeExperiment, OracleEngine
    n, c = logits.shape
    ds = GL.G.IndexDataset(n, c)
    net = GL.G.LookupNet(logits, emb)
    args = dict(early_stop_patience=0, n_epoch=1, world_size=1, model="SSLResNet18", freeze_feature=True,
                ckpt_path=tempfile.mkdtemp(prefix="dropin_"), exp_name="d", subset_labeled=None, subset_unlabeled=None,
                partitions=1)
    args.update(kw)
    s = cls(ds, ds, net, {"loader_te_args": {"batch_size": bs, "num_workers": 0}}, np.array(ev), FakeExperiment(), None, **args)
    s.feature_net = s.net            # what the reference's init_network_weights does (strategy.py:198)
    s.set_engine(OracleEngine())
    if len(lab):
        s.update(np.array(lab), len(lab))
    return s


CASES = GL.DROP_IN_CASES


@pytest.mark.parametrize("name,kw,budget", CASES)
def test_drop_in_classes_on_the_reference_strategy_return_the_reference_picks(ref, name, kw, budget):
    case = CASES.index((name, kw, budget))
    logits, emb, ev, lab = GL.drop_in_inputs()
    mine = _build(ref["accel"][name], logits, emb, ev, lab, 64, **kw)
    # the accelerated class IS a Strategy of the base it was bound to: training, checkpointing, update() are the base's own
    assert isinstance(mine, ref["base"]) and ref["base"] in type(mine).__mro__
    assert type(mine).train is ref["base"].train and type(mine).update is ref["base"].update
    np.random.seed(9)
    got, got_cost = mine.query(budget)
    want, want_cost = ref["gold"][f"dropin{case}_idx"].tolist(), float(ref["gold"][f"dropin{case}_cost"])
    assert [int(i) for i in got] == want and got_cost == want_cost
    # the consumer of query()'s return: update() accepts it (asserts not-yet-labeled, strategy.py:470)
    mine.update(got, got_cost)
    assert mine.idxs_lb[np.asarray(got, dtype=np.int64)].all()
