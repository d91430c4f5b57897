"""The oracle against the reference on fresh random inputs (beyond the committed golden fixtures).

The reference's results on these seeded inputs were produced by running the reference itself
(tests/golden/make_golden_live.py) and are replayed from tests/golden/reference_golden_live.npz; float arrays the
reference returned are compared through their SHA-256 digests, i.e. bit for bit.  Every comparison is exact: the
oracle runs the same torch-CPU / NumPy arithmetic in the same order."""
import os

import numpy as np
import pytest
import torch

from helpers import digest
from oracle import al_oracle as O

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def ref():
    return dict(np.load(os.path.join(GOLD, "reference_golden_live.npz")))


def pool(rng, n, n_eval, n_lab):
    ev = rng.choice(n, size=n_eval, replace=False)
    rest = np.setdiff1d(np.arange(n), ev)
    lab = rng.choice(rest, size=n_lab, replace=False)
    lb = np.zeros(n, dtype=bool)
    lb[lab] = True
    return ev, lab, lb


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_margin_query(ref, seed):
    rng = np.random.default_rng(seed)
    torch.manual_seed(seed)
    n, c = 300 + 17 * seed, (10, 100, 37)[seed]
    ev, lab, lb = pool(rng, n, 20, 40)
    logits = torch.randn(n, c) * 3
    idx, cost = ref[f"margin{seed}_idx"].tolist(), float(ref[f"margin{seed}_cost"])
    avail = O.available_query_idxs(lb, ev, shuffle=False)
    mine, mcost = O.uncertainty_query(logits[avail], avail, 50.0, O.MODE_MARGIN)
    assert mine == idx and mcost == cost


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_pairwise_and_both_coreset_modes(ref, seed):
    rng = np.random.default_rng(10 + seed)
    torch.manual_seed(10 + seed)
    m, d = 200 + 31 * seed, (16, 48, 7)[seed]
    feat = torch.relu(torch.randn(m, d))
    ind = np.zeros(m, dtype=bool)
    ind[rng.choice(m, size=25, replace=False)] = True
    d2 = O.pairwise_l2_dist(feat)
    assert digest(d2) == str(ref[f"coreset{seed}_d2"])          # == the reference's get_pairwise_l2_dist, bit for bit
    greedy = ref[f"coreset{seed}_greedy"].tolist()
    assert O.coreset(d2, ind, 30, randomize=False) == greedy
    assert O.coreset_streaming(feat, ind, 30) == greedy
    want = ref[f"coreset{seed}_sampled"].tolist()
    np.random.seed(seed)
    assert O.coreset(d2, ind, 30, randomize=True) == want
    np.random.seed(seed)                                      # the O(N)-memory form with NumPy-exact sampling arithmetic
    assert O.coreset_streaming(feat, ind, 30, randomize=True) == want
    none = np.zeros(m, dtype=bool)                            # cold start: minimax centre / uniform draw
    assert O.coreset(d2, none, 4, randomize=False) == ref[f"coreset{seed}_cold"].tolist()


@pytest.mark.parametrize("seed", [0, 1])
def test_gradient_embeddings(ref, seed):
    torch.manual_seed(20 + seed)
    n, c, d, bs = (45, 70)[seed], (10, 24)[seed], (12, 40)[seed], (16, 32)[seed]
    lg, h = torch.randn(n, c) * 3, torch.relu(torch.randn(n, d))
    for pooled in (False, True):
        got = O.gradient_embeddings(lg, h, bs, use_adaptive_pool=pooled)
        assert digest(got) == str(ref[f"grad{seed}_emb_{int(pooled)}"])


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_mase_and_base(ref, seed):
    rng = np.random.default_rng(30 + seed)
    torch.manual_seed(30 + seed)
    n, m, c, bs, budget = 260, (8, 24, 16)[seed], (5, 12, 40)[seed], 64, 36
    ev, lab, lb = pool(rng, n, 15, 30)
    # + rand: no all-zero rows -> no exactly equal margins (the reference's torch.sort is not stable on ties)
    emb, w, b = torch.relu(torch.randn(n, m)) + 0.05 * torch.rand(n, m), torch.randn(c, m) * 0.5, torch.randn(c) * 0.1
    avail = O.available_query_idxs(lb, ev, shuffle=False)
    k = f"mase{seed}_"
    omm, opc, opred = O.mase_margins(emb[avail], w, b, bs)
    assert digest(omm) == str(ref[k + "mm"]) and digest(opc) == str(ref[k + "pc"]) and digest(opred) == str(ref[k + "pred"])
    assert O.mase_query(omm, avail, float(budget))[0] == ref[k + "MASESampler"].tolist()
    assert avail[O.base_select(omm, opc, opred, budget, c)].tolist() == ref[k + "BASESampler"].tolist()


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_balancing(ref, seed):
    rng = np.random.default_rng(40 + seed)
    torch.manual_seed(40 + seed)
    n, m, c, budget = 240, 10, (4, 6, 3)[seed], (30, 24, 40)[seed]
    probs = np.array([0.5, 0.25, 0.15, 0.05, 0.03, 0.02][:c])
    ys = rng.choice(c, size=n, p=probs / probs.sum())
    emb = torch.relu(torch.randn(c, m)[torch.from_numpy(ys)] * 2 + torch.randn(n, m))
    ev, lab, lb = pool(rng, n, 12, (40, 25, 60)[seed])
    idx, cost = ref[f"bal{seed}_idx"].tolist(), float(ref[f"bal{seed}_cost"])
    avail = ~lb
    avail[ev] = False
    np.random.seed(seed)
    mine, mcost = O.balancing_query(emb, torch.from_numpy(ys), avail, lb, float(budget), c)
    assert mine == idx and mcost == cost
