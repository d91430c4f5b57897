"""K3 (min-distance contraction) and K4/K5 (selection loop) on the GPU, through the C ABI."""
import numpy as np
import pytest
import torch

from oracle import al_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from active_learning_b200.engine import Engine
    return Engine()


def _split(feat, ind):
    cand, lab = np.flatnonzero(~ind), np.flatnonzero(ind)
    return cand, lab, feat[cand].cuda(), feat[lab].cuda()


def _run(eng, feat, ind, b, randomize=False, uniforms=None, variant=0, first=None, factors=None):
    """Reference-shaped call: dense rows `feat`, boolean labeled indicator -> picks as rows of feat.
    The persistent loop's D^2 draw (variant 3) is run twice -- certified fast path first (default) and exact
    NumPy-tree machinery only -- and both must give the same list."""
    if randomize and variant == 3:
        try:
            eng.set_option("d2_fast_path", 0)
            exact = _run_once(eng, feat, ind, b, randomize, uniforms, variant, first, factors)
        finally:
            eng.set_option("d2_fast_path", 1)
        fast = _run_once(eng, feat, ind, b, randomize, uniforms, variant, first, factors)
        assert fast == exact, "certified fast path and exact path disagree"
        return fast
    return _run_once(eng, feat, ind, b, randomize, uniforms, variant, first, factors)


def _run_once(eng, feat, ind, b, randomize=False, uniforms=None, variant=0, first=None, factors=None):
    cand, lab, X, Y = _split(feat, ind)
    xn = eng.row_norm2(X)
    XA = YA = xan = yan = None
    if factors is not None:
        XA, YA = factors[cand].cuda(), factors[lab].cuda()
        xan = eng.row_norm2(XA)
        yan = eng.row_norm2(YA) if len(lab) else None
    mind = torch.full((len(cand),), float("inf"), device="cuda")
    if len(lab):
        eng.min_dist(X, xn, Y, eng.row_norm2(Y), XA, xan, YA, yan, out=mind)
    picks = eng.greedy_select(X, xn, mind, [0, len(cand)], [b], a=XA, an=xan,
                              uniforms=uniforms if randomize else None,
                              vpos=torch.as_tensor(cand.astype(np.int32)).cuda() if randomize else None,
                              full_n=[len(ind)] if randomize else None,
                              first_pick=[first] if first is not None else None, variant=variant)
    return cand[picks].tolist()


def _assert_prefix_parity(got, ref, feat, ind, randomize):
    """Float fixtures: identical picks expected; if they differ, the first divergence must be a
    near-tie of the oracle's own running min-distances (gap below fp32 noise of n_i + n_j - 2dot)."""
    if got == ref:
        return
    k = next(i for i, (g, r) in enumerate(zip(got, ref)) if g != r)
    assert not randomize, f"D^2-sampling picks diverge at step {k}"
    lab = ind.copy()
    lab[ref[:k]] = True
    d2 = O.pairwise_l2_dist(feat)
    mind = d2[:, lab].min(dim=1).values
    gap = abs(float(mind[got[k]] - mind[ref[k]]))
    scale = float(feat.square().sum(1).max()) * 2
    assert gap <= 1e-5 * scale, f"step {k}: gap {gap} is not a near-tie (scale {scale})"


# ------------------------------------------------------------------------------------------- K3
@pytest.mark.parametrize("n,m,d", [(300, 45, 64), (129, 257, 36), (1000, 1, 2048), (1, 1000, 512), (513, 700, 2048)])
def test_min_dist_exact_on_integer_rows(eng, n, m, d):
    rng = np.random.default_rng(n + m + d)
    x = torch.from_numpy(rng.integers(-1, 2, size=(n, d)).astype(np.float32))
    y = torch.from_numpy(rng.integers(-1, 2, size=(m, d)).astype(np.float32))
    xn, yn = x.square().sum(1), y.square().sum(1)
    d2 = (xn[:, None] + yn[None, :]) - 2 * (x @ y.T)
    got = eng.min_dist(x.cuda(), xn.cuda(), y.cuda(), yn.cuda()).cpu()
    assert torch.equal(got, d2.min(1).values)
    got = eng.min_dist(x.cuda(), xn.cuda(), y.cuda(), yn.cuda(), reduce_max=True).cpu()
    assert torch.equal(got, d2.max(1).values)
    # accumulate over column chunks == one shot
    out = torch.full((n,), float("inf"), device="cuda")
    for lo in range(0, m, 100):
        eng.min_dist(x.cuda(), xn.cuda(), y[lo:lo + 100].cuda(), yn[lo:lo + 100].cuda(), out=out, accumulate=True)
    assert torch.equal(out.cpu(), d2.min(1).values)


def test_min_dist_float_and_factored(eng):
    torch.manual_seed(0)
    x, y = torch.relu(torch.randn(700, 2048)), torch.relu(torch.randn(333, 2048))
    xn, yn = x.square().sum(1), y.square().sum(1)
    ref = ((xn[:, None] + yn[None, :]) - 2 * (x.double() @ y.double().T)).min(1).values
    got = eng.min_dist(x.cuda(), eng.row_norm2(x.cuda()), y.cuda(), eng.row_norm2(y.cuda())).cpu().double()
    assert ((got - ref).abs() <= 1e-5 * (xn.max() + yn.max()).double()).all()
    # factored rows against the materialised rank-1 embedding (fp64 truth)
    rng = np.random.default_rng(1)
    xa, ya = torch.randn(200, 40) * 0.05, torch.randn(90, 40) * 0.05
    xh, yh = torch.relu(torch.randn(200, 64)), torch.relu(torch.randn(90, 64))
    gx = (xa[:, :, None] * xh[:, None, :]).reshape(200, -1).double()
    gy = (ya[:, :, None] * yh[:, None, :]).reshape(90, -1).double()
    ref = torch.cdist(gx, gy).square().min(1).values
    c = lambda t: t.cuda()
    got = eng.min_dist(c(xh), eng.row_norm2(c(xh)), c(yh), eng.row_norm2(c(yh)),
                       c(xa), eng.row_norm2(c(xa)), c(ya), eng.row_norm2(c(ya))).cpu().double()
    scale = gx.square().sum(1).max() + gy.square().sum(1).max()
    assert ((got - ref).abs() <= 1e-5 * scale).all()
    # factored, exact integers
    xa = torch.from_numpy(rng.integers(-1, 2, size=(150, 8)).astype(np.float32))
    xh = torch.from_numpy(rng.integers(-1, 2, size=(150, 16)).astype(np.float32))
    g = (xa[:, :, None] * xh[:, None, :]).reshape(150, -1)
    d2 = O.pairwise_l2_dist(g)
    got = eng.min_dist(c(xh[:100]), eng.row_norm2(c(xh[:100])), c(xh[100:]), eng.row_norm2(c(xh[100:])),
                       c(xa[:100]), eng.row_norm2(c(xa[:100])), c(xa[100:]), eng.row_norm2(c(xa[100:]))).cpu()
    assert torch.equal(got, d2[:100, 100:].min(1).values)


@pytest.mark.parametrize("n,m,d,c", [(300, 700, 96, 0), (1000, 1000, 2048, 0), (777, 1313, 516, 0),
                                     (500, 600, 64, 40), (640, 900, 2048, 1000)])
def test_min_dist_tensor_core_path(eng, n, m, d, c):
    """wgmma 3xTF32 contraction (k3_impl=2): bit-identical to fp32 on integer rows (lo == 0), within
    1e-5 * (|x|^2 + |y|^2) of the fp64 truth on float rows; min and max epilogues; accumulate."""
    rng = np.random.default_rng(n + m + d + c)
    cu = lambda t: t.cuda()
    try:
        eng.set_option("k3_impl", 2)
        for ints in (True, False):
            if ints:
                x = torch.from_numpy(rng.integers(-1, 2, size=(n, d)).astype(np.float32))
                y = torch.from_numpy(rng.integers(-1, 2, size=(m, d)).astype(np.float32))
                xa = torch.from_numpy(rng.integers(-1, 2, size=(n, max(c, 1))).astype(np.float32))
                ya = torch.from_numpy(rng.integers(-1, 2, size=(m, max(c, 1))).astype(np.float32))
            else:
                x, y = torch.relu(torch.randn(n, d)), torch.relu(torch.randn(m, d))
                xa, ya = torch.randn(n, max(c, 1)) * 0.05, torch.randn(m, max(c, 1)) * 0.05
            dot = x.double() @ y.double().T
            nx, ny = x.double().square().sum(1), y.double().square().sum(1)
            args = [cu(x), eng.row_norm2(cu(x)), cu(y), eng.row_norm2(cu(y))]
            if c:
                dot = dot * (xa.double() @ ya.double().T)
                nx, ny = nx * xa.double().square().sum(1), ny * ya.double().square().sum(1)
                args += [cu(xa), eng.row_norm2(cu(xa)), cu(ya), eng.row_norm2(cu(ya))]
            d2 = (nx[:, None] + ny[None, :]) - 2 * dot
            tol = 0.0 if ints else 1e-5 * float(nx.max() + ny.max())
            got = eng.min_dist(*args).cpu().double()
            assert (got - d2.min(1).values).abs().max() <= tol
            got = eng.min_dist(*args, reduce_max=True).cpu().double()
            assert (got - d2.max(1).values).abs().max() <= tol
        out = torch.full((n,), float("inf"), device="cuda")      # accumulate over column chunks
        half = m // 2
        for sl in (slice(0, half), slice(half, m)):
            a2 = [args[0], args[1], args[2][sl], args[3][sl]]
            if c:
                a2 += [args[4], args[5], args[6][sl], args[7][sl]]
            eng.min_dist(*a2, out=out, accumulate=True)
        assert (out.cpu().double() - d2.min(1).values).abs().max() <= tol
    finally:
        eng.set_option("k3_impl", 0)


# ------------------------------------------------------------------------------------------- K4 / K5 vs golden
@pytest.mark.parametrize("variant", [1, 2, 3])
@pytest.mark.parametrize("tag", ["int", "f32"])
def test_greedy_matches_reference_golden(eng, gold, tag, variant):
    feat, ind = torch.from_numpy(gold[f"cs_{tag}_feat"]), gold["cs_indicator"]
    got = _run(eng, feat, ind, 40, variant=variant)
    ref = gold[f"cs_{tag}_greedy"].tolist()
    if tag == "int":
        assert got == ref
    else:
        _assert_prefix_parity(got, ref, feat, ind, False)


@pytest.mark.parametrize("variant", [1, 2, 3])
@pytest.mark.parametrize("tag", ["int", "f32"])
def test_d2_sampling_matches_reference_golden(eng, gold, tag, variant):
    feat, ind = torch.from_numpy(gold[f"cs_{tag}_feat"]), gold["cs_indicator"]
    np.random.seed(11)
    us = np.random.random_sample(40)
    got = _run(eng, feat, ind, 40, randomize=True, uniforms=us, variant=variant)
    assert got == gold[f"cs_{tag}_d2sample"].tolist()


def test_cold_start_matches_reference_golden(eng, gold):
    for tag in ("int", "f32"):
        feat = torch.from_numpy(gold[f"cs_{tag}_feat"])
        none = np.zeros(len(feat), dtype=bool)
        X = feat.cuda()
        xn = eng.row_norm2(X)
        q0 = eng.argmin(eng.min_dist(X, xn, X, xn, reduce_max=True))          # minimax centre
        assert q0 == int(gold[f"cs_{tag}_greedy_cold"][0])
        for variant in (2, 3):
            assert _run(eng, feat, none, 6, first=q0, variant=variant) == gold[f"cs_{tag}_greedy_cold"].tolist()
        np.random.seed(12)
        q0 = int(np.random.choice(len(feat)))
        us = np.zeros(6)
        us[1:] = np.random.random_sample(5)
        for variant in (2, 3):
            assert _run(eng, feat, none, 6, randomize=True, uniforms=us, first=q0, variant=variant) == \
                gold[f"cs_{tag}_d2sample_cold"].tolist()


def test_nan_retry_branch_matches_reference_golden(eng, gold):
    """All candidates duplicate labeled rows: sum(prob) == 0 -> NaN -> `+= 1e-5` retry."""
    feat, ind = torch.from_numpy(gold["cs_dup_feat"]), gold["cs_dup_indicator"]
    np.random.seed(13)
    us = np.random.random_sample(5)
    for variant in (1, 2, 3):
        assert _run(eng, feat, ind, 5, randomize=True, uniforms=us, variant=variant) == gold["cs_dup_d2sample"].tolist()


# ------------------------------------------------------------------------------------------- larger, vs oracle
@pytest.mark.parametrize("randomize", [False, True])
@pytest.mark.parametrize("d", [512, 2048])
def test_greedy_exact_fixture_medium(eng, randomize, d):
    """P0 ladder rung: integer rows make every fp32 op exact in any order -> identical lists."""
    rng = np.random.default_rng(d + randomize)
    n, l0, b = 6000, 900, 120
    feat = torch.from_numpy(rng.integers(-1, 2, size=(n, d)).astype(np.float32))
    ind = np.zeros(n, dtype=bool)
    ind[rng.choice(n, l0, replace=False)] = True
    us = rng.random(b)
    ref = O.coreset_streaming(feat, ind, b, randomize=randomize, uniforms=us)
    for variant in (1, 2, 3):
        assert _run(eng, feat, ind, b, randomize=randomize, uniforms=us, variant=variant) == ref


def test_d2_sampling_large_tree_exact(eng):
    """Deep NumPy pairwise tree (full array of 60 000 -> 512 leaves, 9 levels, every slice of the 8-CTA
    cluster populated) on an exact-arithmetic fixture: picks must equal the oracle's, factored and dense."""
    rng = np.random.default_rng(77)
    n, l0, b = 52000, 8000, 90
    for c in (0, 8):
        h = torch.from_numpy(rng.integers(-1, 2, size=(n + l0, 32)).astype(np.float32))
        a = torch.from_numpy(rng.integers(-1, 2, size=(n + l0, 8)).astype(np.float32)) if c else None
        ind = np.zeros(n + l0, dtype=bool)
        ind[rng.choice(n + l0, l0, replace=False)] = True
        us = rng.random(b)
        feat = h if a is None else (a[:, :, None] * h[:, None, :]).reshape(n + l0, -1)
        ref = O.coreset_streaming(feat, ind, b, randomize=True, uniforms=us)
        for variant in (2, 3):
            assert _run(eng, h, ind, b, randomize=True, uniforms=us, factors=a, variant=variant) == ref


def test_badge_factored_equals_materialised_reference(eng):
    """K5 on rank-1 factors == the reference's dense path on the materialised a (x) h."""
    rng = np.random.default_rng(9)
    n, c, d, l0, b = 900, 8, 16, 120, 60
    a = torch.from_numpy(rng.integers(-1, 2, size=(n, c)).astype(np.float32))
    h = torch.from_numpy(rng.integers(-1, 2, size=(n, d)).astype(np.float32))
    g = (a[:, :, None] * h[:, None, :]).reshape(n, -1)
    ind = np.zeros(n, dtype=bool)
    ind[rng.choice(n, l0, replace=False)] = True
    d2 = O.pairwise_l2_dist(g)
    np.random.seed(3)
    ref_rand = O.coreset(d2, ind, b, randomize=True)
    np.random.seed(3)
    us = np.random.random_sample(b)
    for variant in (1, 2, 3):
        assert _run(eng, h, ind, b, randomize=True, uniforms=us, factors=a, variant=variant) == ref_rand
        assert _run(eng, h, ind, b, factors=a, variant=variant) == O.coreset(d2, ind, b)


def test_partitions_are_a_batch_dimension(eng):
    """One batched launch over P partitions == P separate runs (argmax and sampling)."""
    rng = np.random.default_rng(21)
    sizes, labs, budgets = [700, 1301, 64, 999], [80, 0, 10, 200], [30, 29, 5, 30]
    feats = [torch.relu(torch.randn(s + l, 512, generator=torch.Generator().manual_seed(i)))
             for i, (s, l) in enumerate(zip(sizes, labs))]
    for randomize in (False, True):
        us = [rng.random(b) for b in budgets]
        solo, X, mind, vpos, first = [], [], [], [], []
        for p, f in enumerate(feats):
            ind = np.zeros(len(f), dtype=bool)
            ind[:labs[p]] = True
            fp = None
            if labs[p] == 0:
                fp = 17
            solo.append(_run(eng, f, ind, budgets[p], randomize=randomize, uniforms=us[p], first=fp))
            Xp = f[labs[p]:].cuda()
            X.append(Xp)
            m = torch.full((sizes[p],), float("inf"), device="cuda")
            if labs[p]:
                Y = f[:labs[p]].cuda()
                eng.min_dist(Xp, eng.row_norm2(Xp), Y, eng.row_norm2(Y), out=m)
            mind.append(m)
            vpos.append(labs[p] + np.arange(sizes[p]))
            first.append(-1 if labs[p] else 17 + int(np.sum(sizes[:p])))
        Xall = torch.cat(X)
        off = np.concatenate(([0], np.cumsum(sizes))).astype(np.int32)
        for variant in (2, 3):
            picks = eng.greedy_select(Xall, eng.row_norm2(Xall), torch.cat(mind).clone(), off, budgets,
                                      uniforms=np.concatenate(us) if randomize else None,
                                      vpos=torch.as_tensor(np.concatenate(vpos).astype(np.int32)).cuda() if randomize else None,
                                      full_n=[s + l for s, l in zip(sizes, labs)] if randomize else None,
                                      first_pick=first, variant=variant)
            at = 0
            for p in range(4):
                got = (picks[at:at + budgets[p]] - off[p] + labs[p]).tolist()
                assert got == solo[p], (randomize, p, variant)
                at += budgets[p]


def test_full_size_coreset_properties(eng):
    """BASELINE config 2 shape: 80k candidates x 2048, 50k labeled (integers -> exact), B = 150.
    The oracle cannot run this size; check against an exact torch-on-GPU restatement of the same
    recurrence, plus uniqueness and the final running-min invariant."""
    g = torch.Generator(device="cuda").manual_seed(0)
    X = torch.randint(-1, 2, (80000, 2048), device="cuda", generator=g).float()
    Y = torch.randint(-1, 2, (50000, 2048), device="cuda", generator=g).float()
    xn, yn = eng.row_norm2(X), eng.row_norm2(Y)
    mind = eng.min_dist(X, xn, Y, yn)
    ref = torch.full((80000,), float("inf"), device="cuda")
    for lo in range(0, 50000, 5000):
        d2 = (xn[:, None] + yn[None, lo:lo + 5000]) - 2 * (X @ Y[lo:lo + 5000].T)
        ref = torch.minimum(ref, d2.min(1).values)
    assert torch.equal(mind, ref)
    b = 150
    m0 = mind.clone()
    picks1 = eng.greedy_select(X, xn, mind, [0, 80000], [b], variant=1)
    picks2 = eng.greedy_select(X, xn, m0.clone(), [0, 80000], [b], variant=2)
    picks3 = eng.greedy_select(X, xn, m0.clone(), [0, 80000], [b], variant=3)
    assert picks1.tolist() == picks2.tolist() == picks3.tolist() and len(set(picks1.tolist())) == b
    m = m0.clone()
    for t in range(b):
        mm = m.clone()
        mm[torch.as_tensor(picks1[:t].astype(np.int64), device="cuda")] = float("-inf")
        q = int(torch.argmax(mm))                    # first max == lowest row on ties
        assert q == int(picks1[t]), t
        m = torch.minimum(m, (xn + xn[q]) - 2 * (X @ X[q]))


# ------------------------------------------------------------------------------------------- BASELINE config 4 dimensions
@pytest.mark.parametrize("randomize", [False, True])
def test_factored_step_at_north_star_dimensions_exact(eng, randomize):
    """The K5 / K4 step on rank-1 factors at C = 1000, D = 2048 (BASELINE config 4: 12 192-byte rows, 2 rows per
    24 KB tile -- a different tile geometry from the small factored fixtures) on an exact-arithmetic fixture:
    N = 6 000 rows, 900 labeled, 120 picks, against the oracle's factored streaming form (pinned to the
    materialised reference path by tests/test_oracle_golden.py).  Every variant, identical lists."""
    rng = np.random.default_rng(41 + randomize)
    n, l0, b, c, d = 6000, 900, 120, 1000, 2048
    h = torch.from_numpy(rng.integers(-1, 2, size=(n, d)).astype(np.float32))
    a = torch.from_numpy(rng.integers(-1, 2, size=(n, c)).astype(np.float32))
    ind = np.zeros(n, dtype=bool)
    ind[rng.choice(n, l0, replace=False)] = True
    us = rng.random(b)
    ref = O.coreset_streaming(h, ind, b, randomize=randomize, uniforms=us, factors=a)
    assert len(set(ref)) == b
    for variant in (1, 2, 3):
        assert _run(eng, h, ind, b, randomize=randomize, uniforms=us, factors=a, variant=variant) == ref, variant


@pytest.mark.parametrize("randomize", [False, True])
@pytest.mark.parametrize("c", [0, 1000])
def test_float_fixture_d2048_with_gap_certificate(eng, randomize, c):
    """SURVEY.md section 7 rung P1: float rows at d = 2048 (dense) and at C = 1000 x D = 2048 (factored).  The GPU
    sums the dot products in a different order than MKL, so its distances differ from the oracle's in the last bits;
    the oracle records, per step, how far its own decision was from flipping (arg-max: gap to the runner-up;
    D^2 draw: distance of u from the nearest cdf breakpoint).  Picks must be identical up to the first step whose
    certificate is below the rounding noise of fl(n_i + n_q - 2 dot) -- and that step, if any, must exist."""
    g = torch.Generator().manual_seed(100 + 2 * c + randomize)
    n, l0, b, d = 4000, 600, 80, 2048
    h = torch.relu(torch.randn(n, d, generator=g))
    a = None
    if c:
        z = torch.randn(n, c, generator=g) * 3
        a = O.badge_factors(z, 128)
    ind = np.zeros(n, dtype=bool)
    ind[torch.randperm(n, generator=g)[:l0].numpy()] = True
    us = np.random.default_rng(c + randomize).random(b)
    cert = []
    ref = O.coreset_streaming(h, ind, b, randomize=randomize, uniforms=us, factors=a, certificate=cert)
    nsq = h.square().sum(1) * (a.square().sum(1) if a is not None else 1.0)
    noise = 4e-6 * float(nsq.max()) * 2                     # a few ulps of n_i + n_q
    for variant in (2, 3):
        got = _run(eng, h, ind, b, randomize=randomize, uniforms=us, factors=a, variant=variant)
        if got == ref:
            continue
        k = next(i for i, (x, y) in enumerate(zip(got, ref)) if x != y)
        thr = noise if not randomize else noise / float(nsq.mean())     # cdf units: relative to the total mass
        assert cert[k] <= thr, f"variant {variant}: picks diverge at step {k} whose certificate {cert[k]} > {thr}"
