"""ALFAMixSampler without a GPU: the collapse of the paper's mixing to one threshold per row against a literal restatement,
t* against a sweep over t, the anchors' empty-class rule, the cap walk, and the sampler's host logic (the all-candidates
branch, the fill, the RNG draw order, a zero budget, no labeled rows, alpha_step) through a fake engine built on the
oracle."""
import math

import numpy as np
import pytest
import torch

import alfamix_oracle as AO
import typiclust_oracle as T
from helpers import HeadNet, LabeledIndexDataset, OracleEngine, make_strategy


def _head_fixture(seed, n, c, d):
    """Integer embeddings and head: every logit is exact in fp32 and fp64, in any order."""
    rng = np.random.default_rng(seed)
    z = rng.integers(-3, 4, size=(n, d)).astype(np.float32)
    w = rng.integers(-2, 3, size=(c, d)).astype(np.float32)
    b = rng.integers(-2, 3, size=c).astype(np.float32)
    return rng, z, w, b, (z.astype(np.float64) @ w.T.astype(np.float64) + b).astype(np.float32)


@pytest.mark.parametrize("seed", range(4))
def test_the_threshold_equals_the_papers_mixing_at_every_cap(seed):
    n, c, d = 160, 6, 12
    rng, z, w, b, logits = _head_fixture(seed, n, c, d)
    anc = (rng.normal(size=(c, d)) * 2.0).astype(np.float32)
    assert (anc[None, :, :] != z[:, None, :]).all()                     # no zero coordinate of a - z
    rho = AO.rho(logits, z, anc, w)
    kappa = np.arange(1, 33) * AO.ALPHA_STEP
    fin = np.isfinite(rho)
    assert (np.abs(rho[fin, None] - kappa[None, :]) > 1e-9 * kappa[None, :]).all()   # no rho at rounding of a cap
    flipped = 0
    for k in kappa:
        want = AO.literal_flips(z, anc, w, b, k / math.sqrt(d))
        assert (want == (rho < k)).all(), k
        flipped += int(want.sum())
    assert 0 < flipped < n * len(kappa)                                 # both outcomes occur


def test_tstar_equals_a_sweep_over_t():
    rng, z, w, b, logits = _head_fixture(7, 40, 5, 8)
    logits = logits + rng.normal(size=logits.shape).astype(np.float32) * 0.25
    y, _, wv, s2 = AO.head_terms(logits, w)
    t = AO.tstar(logits, y, wv, s2)
    for u in range(len(z)):
        if not np.isfinite(t[u]):
            continue
        grid = np.linspace(0.0, 2.0 * t[u] + 1e-6, 20001)
        mixed = logits[u].astype(np.float64)[None, :] + grid[:, None] * (wv[u] / math.sqrt(s2[u]))[None, :]
        flips = np.flatnonzero(mixed.argmax(axis=1) != y[u])
        assert len(flips)
        step = grid[1] - grid[0]
        assert grid[flips[0]] - step <= t[u] <= grid[flips[0]] + 1e-12


def test_anchors_take_the_mean_of_all_labeled_rows_for_an_empty_class():
    rng = np.random.default_rng(3)
    emb = rng.normal(size=(30, 8)).astype(np.float32)
    labels = rng.choice([0, 2, 3], size=30)
    anc = AO.anchors(emb, labels, 5)
    glob = (np.cumsum(emb.astype(np.float64), axis=0)[-1] / 30).astype(np.float32)
    for c in range(5):
        rows = np.flatnonzero(labels == c)
        want = glob if not len(rows) else (np.cumsum(emb[rows].astype(np.float64), axis=0)[-1] / len(rows)).astype(np.float32)
        assert (anc[c].view(np.uint32) == want.view(np.uint32)).all(), c


@pytest.mark.parametrize("step", [2.0 ** -5, 0.1, 0.3, 1.0, 1e-3])
def test_the_samplers_cap_walk_equals_the_walk_one_cap_at_a_time(step):
    from active_learning_b200.query_strategies.alfamix import cap_walk
    rng = np.random.default_rng(int(step * 1e4))
    for _ in range(40):
        n = int(rng.integers(1, 300))
        rho = rng.uniform(0, 1.3, size=n)
        rho[rng.random(n) < 0.1] = np.inf
        grid = np.arange(1, math.ceil(1 / step) + 1) * step
        tie = rng.random(n) < 0.2                                       # rho exactly on a cap
        rho[tie] = rng.choice(grid, int(tie.sum()))
        for budget in (1, n // 3, n - 1, n, n + 5):
            want = AO.cap_walk(rho, budget, step)
            assert cap_walk(rho, budget, step).tolist() == want.tolist()
            j = math.ceil(1 / step)
            for jj in range(1, j + 1):
                if (rho < jj * step).sum() > budget:
                    j = jj
                    break
            assert want.tolist() == np.flatnonzero(rho < j * step).tolist()


class ALFAEngine(OracleEngine):
    """The oracle engine plus the ALFA-Mix calls by the NumPy statement; records what ran."""

    def __init__(self):
        self.calls = []

    def kmeans_update(self, x, labels, centres):
        centres[:] = torch.from_numpy(T.update(x.numpy(), labels.numpy().astype(np.int64), centres.numpy()))
        return centres

    def alfamix_rho(self, logits, emb, anchors, weight):
        self.calls.append("rho")
        return torch.from_numpy(AO.rho(logits.numpy(), emb.numpy(), anchors.numpy(), weight.numpy()))

    def normalize(self, x):
        return torch.from_numpy(T.normalize(x.numpy()))

    def kmeans(self, xhat, first, unif, k, max_iter):
        self.calls.append("kmeans")
        x = xhat.numpy()
        seeds = T.seed(x, first, unif, k)
        labels, centres, it = T.lloyd(x, x[seeds].copy(), max_iter)
        return torch.from_numpy(labels.astype(np.int32)), torch.from_numpy(centres), it, seeds

    def kmeans_nearest(self, xhat, labels, centres):
        return AO.nearest(xhat.numpy(), labels.numpy(), centres.numpy())


def _sampler(n=240, c=5, d=8, seed=2, n_lab=30, engine=None, **kw):
    rng = np.random.default_rng(seed)
    emb = rng.integers(-3, 4, size=(n, d)).astype(np.float32)
    w = rng.integers(-2, 3, size=(c, d)).astype(np.float32)
    bias = rng.integers(-2, 3, size=c).astype(np.float32)
    ys = rng.integers(0, c, size=n)
    net = HeadNet(torch.from_numpy(emb), torch.from_numpy(w), torch.from_numpy(bias))
    ev = rng.choice(n, 12, replace=False)
    lab = rng.choice(np.setdiff1d(np.arange(n), ev), n_lab, replace=False) if n_lab else []
    s = make_strategy("ALFAMixSampler", None, None, ev, lab, 32, engine=engine or ALFAEngine(), net=net,
                      dataset=LabeledIndexDataset(ys, c), **kw)
    return s, emb, w, ys


def _expected(s, emb, w, ys, budget, step=AO.ALPHA_STEP):
    union = np.asarray(s.get_idxs_for_coreset(), dtype=np.int64)
    is_lab = s.already_labeled_idxs(boolean=True)[union]
    avail = s.available_query_idxs(boolean=True)[union]
    with torch.no_grad():
        logits = s.net.linear(torch.from_numpy(emb)).numpy()
    return union[AO.query_positions(emb[union], logits[union], w, ys[union][is_lab], is_lab, avail, budget, step)].tolist()


@pytest.mark.parametrize("budget,step,branch", [(20, 2.0 ** -5, "kmeans"), (60, 2.0 ** -5, "kmeans"),
                                                (190, 0.5, "all"), (10 ** 6, 2.0 ** -5, "all")])
def test_query_equals_the_oracle_and_its_draws(budget, step, branch):
    s, emb, w, ys = _sampler(alpha_step=step)
    eng = s.get_engine()
    np.random.seed(21)
    got, k = s.query(budget)
    after = np.random.get_state()
    np.random.seed(21)
    want = _expected(s, emb, w, ys, budget, step)
    assert got == want and k == len(want) == min(budget, int(s.available_query_idxs(boolean=True).sum()))
    assert (np.random.get_state()[1] == after[1]).all() and np.random.get_state()[2] == after[2]
    assert len(set(got)) == k and not s.idxs_lb[got].any()
    assert ("kmeans" in eng.calls) == (branch == "kmeans")


def test_the_draws_in_order_shuffles_seeding_fill():
    """With k-means, replayed draw by draw: two permutations, choice(|cand|), K - 1 uniforms, then the fill's choice over
    the available, unpicked positions if the clusters leave a remainder."""
    s, emb, w, ys = _sampler(n=400, n_lab=40, c=4)
    budget = 60
    np.random.seed(5)
    got, _ = s.query(budget)
    after = np.random.get_state()
    np.random.seed(5)
    union = np.asarray(s.get_idxs_for_coreset(), dtype=np.int64)          # draws 1 and 2
    is_lab = s.already_labeled_idxs(boolean=True)[union]
    avail = s.available_query_idxs(boolean=True)[union]
    e = emb[union]
    with torch.no_grad():
        logits = s.net.linear(torch.from_numpy(e)).numpy()
    cand = np.flatnonzero(avail)
    sel = cand[AO.cap_walk(AO.rho(logits[cand], e[cand], AO.anchors(e[is_lab], ys[union][is_lab], 4), w), budget)]
    assert len(sel) > budget
    first = int(np.random.choice(len(sel)))                                # draw 3
    unif = np.random.random_sample(budget - 1)                             # draw 4
    xhat = T.normalize(e[sel])
    labels, centres, _ = T.lloyd(xhat, xhat[T.seed(xhat, first, unif, budget)].copy())
    near = AO.nearest(xhat, labels, centres)
    picks = sel[near[near >= 0]]
    if len(picks) < budget:                                                # empty clusters leave a remainder
        free = avail.copy()
        free[picks] = False
        picks = np.concatenate([picks, np.random.choice(np.flatnonzero(free), budget - len(picks), replace=False)])
    assert got == union[picks].tolist()
    assert (np.random.get_state()[1] == after[1]).all() and np.random.get_state()[2] == after[2]


def test_zero_budget_no_labeled_rows_and_alpha_step():
    for n_lab in (30, 0):
        s, *_ = _sampler(n_lab=n_lab)
        for budget in (0, -3):
            np.random.seed(5)
            assert s.query(budget) == ([], 0)
            state = np.random.get_state()
            np.random.seed(5)
            s.get_idxs_for_coreset()
            assert (np.random.get_state()[1] == state[1]).all() and np.random.get_state()[2] == state[2]
        assert s.get_engine().calls == []
    with pytest.raises(ValueError, match="ALFAMixSampler needs labeled rows"):
        s.query(10)
    for bad in (0.0, -0.5, 1.5, float("nan"), float("inf"), "x", None):
        with pytest.raises(ValueError, match="alpha_step"):
            _sampler(alpha_step=bad)
    assert _sampler(alpha_step=1.0)[0].alpha_step == 1.0
    assert _sampler()[0].alpha_step == 2.0 ** -5


def test_a_net_without_a_linear_head_is_a_clear_error():
    s, *_ = _sampler()
    s.net = s.feature_net = torch.nn.Identity()
    with pytest.raises(AttributeError, match="no `.linear` layer"):
        s.query(10)


def test_dispatch_and_drop_in():
    from active_learning_b200.integration import make_drop_in
    from active_learning_b200.query_strategies.get_strategy import ACCELERATED, get_strategy
    from active_learning_b200.query_strategies.strategy import Strategy
    assert "ALFAMixSampler" in ACCELERATED and get_strategy("ALFAMixSampler").__name__ == "ALFAMixSampler"
    assert "ALFAMixSampler" in make_drop_in(Strategy)
