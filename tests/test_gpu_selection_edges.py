"""K4/K5 (the CoreSet / BADGE selection loop) at the branches chosen from the problem's shape or from the uniform's value:
the certified D^2 fast path next to its margin, CTA segments beyond the 2 048 rows whose masses stay in shared memory,
the `+= 1e-5` retry branch across many CTAs, and variant=0's host-side choice between the persistent loop and the
per-step kernels.  Every test checks that it reached its branch (the variant that ran, rows per CTA, tree leaves,
certificates) and compares the picks with the oracle.  Integer fixtures make every fp32 operation exact."""
import numpy as np
import pytest
import torch

from helpers import BoundaryUniforms
from oracle import al_oracle as O
from test_gpu_greedy import _run

pytestmark = pytest.mark.gpu

PERSIST_MAX_LEAVES = 4096        # alq_greedy_persist.cu kMaxLeaves
ROW_MASS_ROWS = 2048             # a CTA keeps its rows' D^2 masses in shared memory up to this many rows
KEY_ROW_OFFSET = 65535           # the persistent arg-max word holds a 16-bit row offset


@pytest.fixture(scope="module")
def eng():
    from active_learning_b200.engine import Engine
    return Engine()


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _ints(rng, rows, cols):
    return torch.from_numpy(rng.integers(-1, 2, size=(rows, cols)).astype(np.float32))


def _fixture(rng, n, l0, d, c=0):
    """n candidates and l0 labeled rows at random positions of the full array, integer entries in {-1, 0, 1}."""
    h = _ints(rng, n + l0, d)
    a = _ints(rng, n + l0, c) if c else None
    ind = np.zeros(n + l0, dtype=bool)
    ind[rng.choice(n + l0, l0, replace=False)] = True
    return h, a, ind


def _seg_end_positions(ind, grid):
    """Full-array position of the last candidate of each CTA segment: with one partition on one GPU the persistent loop
    gives CTA j the candidate rows [n j / G, n (j + 1) / G)."""
    cand = np.flatnonzero(~ind)
    n = len(cand)
    return cand[[n * (j + 1) // grid - 1 for j in range(grid)]]


def _variant(eng):
    return eng.last_greedy_timing["variant"]


def _raises_then_usable(eng, call, match):
    """`call` must raise the library's AlqError, and the engine must keep working afterwards."""
    from active_learning_b200.engine import AlqError
    with pytest.raises(AlqError, match=match):
        call()
    v = torch.arange(8, dtype=torch.float32, device="cuda")
    assert eng.argmin(v) == 0


# ------------------------------------------------------------------------------------------- A: D^2 draw at its boundaries
@pytest.mark.parametrize("c", [0, 8])
def test_d2_draw_with_uniforms_on_cdf_breakpoints(eng, sms, c):
    """u on, one ulp beside, and 1.0-5e-7 away from cdf breakpoints (including the last position of every CTA segment,
    u = 0 and u = 1 - 2^-53): steps the fast path must hand to the exact path, and steps it decides right next to its
    1.3e-7 margin.  Variant 3 with and without the fast path, and variant 2, all equal the oracle."""
    rng = np.random.default_rng(100 + c)
    n, l0, b = 20000, 2000, 100
    h, a, ind = _fixture(rng, n, l0, 64, c)
    f = BoundaryUniforms(c, seg_end_pos=_seg_end_positions(ind, sms))
    cert = []
    ref = O.coreset_streaming(h, ind, b, randomize=True, uniforms=f, factors=a, certificate=cert)
    assert sum(x < 1e-8 for x in cert) >= 10                  # undecidable by the fast path: the exact path runs
    assert sum(1.3e-7 < x <= 5e-7 for x in cert) >= 10        # decided just outside the margin
    us = np.array(f.us)
    for variant in (3, 2):
        assert _run(eng, h, ind, b, randomize=True, uniforms=us, factors=a, variant=variant, time_steps=True) == ref
        assert _variant(eng) == variant


@pytest.mark.parametrize("c", [0, 8])
def test_persistent_loop_with_cta_segments_beyond_shared_row_masses(eng, sms, c):
    """2 200 rows per CTA: the row masses are not kept in shared memory and the fast path searches the crossing CTA's
    rows in global memory (block_locate).  D^2 with the boundary schedule, and arg-max, equal the oracle."""
    rng = np.random.default_rng(200 + c)
    n, l0, b = 2200 * sms, 200, 100
    h, a, ind = _fixture(rng, n, l0, 8, c)
    assert n // sms > ROW_MASS_ROWS
    assert len(O.pairwise_leaves(n + l0)) <= PERSIST_MAX_LEAVES
    f = BoundaryUniforms(200 + c, seg_end_pos=_seg_end_positions(ind, sms))
    ref = O.coreset_streaming(h, ind, b, randomize=True, uniforms=f, factors=a)
    assert _run(eng, h, ind, b, randomize=True, uniforms=np.array(f.us), factors=a, variant=3, time_steps=True) == ref
    assert _variant(eng) == 3
    ref = O.coreset_streaming(h, ind, b, factors=a)
    assert _run(eng, h, ind, b, factors=a, variant=3, time_steps=True) == ref
    assert _variant(eng) == 3


@pytest.mark.parametrize("variant", [2, 3])
def test_identical_candidates_retry_branch_and_ties_across_ctas(eng, sms, variant):
    """20 000 copies of one row, none of them labeled.  D^2: after the first pick every distance is 0, so every later
    step takes the `+= 1e-5` retry branch (equal to the oracle).  Arg-max: every later step is a tie of all remaining
    rows, resolved to the lowest row across CTA boundaries.  (The oracle, like the reference, lets the picked and the
    labeled rows compete in that tie and re-picks position 0 -- the deliberate deviation of DESIGN.md section 2 -- so
    only its first pick is compared.)"""
    rng = np.random.default_rng(300)
    n, l0, b, d = 20000, 200, 400, 8
    lab = _ints(rng, l0, d)
    lab[lab.sum(1) == d] = 0.0                                # no labeled row equals the candidate row (all ones)
    feat = torch.cat([torch.ones(n, d), lab])
    ind = np.zeros(n + l0, dtype=bool)
    ind[n:] = True
    perm = rng.permutation(n + l0)                            # labeled rows scattered among the candidates
    feat, ind = feat[perm], ind[perm]
    cand = np.flatnonzero(~ind)
    assert b > 2 * (n // sms)                                 # the picks run through three CTA segments or more
    us = rng.random(b)
    with np.errstate(invalid="ignore"):
        ref = O.coreset_streaming(feat, ind, b, randomize=True, uniforms=us)
    assert _run(eng, feat, ind, b, randomize=True, uniforms=us, variant=variant, time_steps=True) == ref
    assert _variant(eng) == variant
    got = _run(eng, feat, ind, b, variant=variant, time_steps=True)
    assert _variant(eng) == variant
    assert got[0] == O.coreset_streaming(feat, ind, 1)[0] == cand[0]
    assert got == cand[:b].tolist()


# ------------------------------------------------------------------------------------------- B: variant=0's choices
def _d2_case(eng, rng, full, b=40, l0=200):
    """One unpartitioned D^2 query over a full array of `full` positions, d = 8 integers."""
    h, _, ind = _fixture(rng, full - l0, l0, 8)
    us = rng.random(b)
    return h, ind, us


@pytest.mark.parametrize("full,leaves,variant", [(524288, 4096, 3), (524289, 4097, 2), (600000, 8192, 2)])
def test_tree_leaf_limit_of_the_persistent_loop(eng, full, leaves, variant):
    rng = np.random.default_rng(full)
    h, ind, us = _d2_case(eng, rng, full)
    assert len(O.pairwise_leaves(full)) == leaves
    if variant != 3:
        _raises_then_usable(eng, lambda: _run(eng, h, ind, len(us), randomize=True, uniforms=us, variant=3),
                            "persistent loop does not fit")
    ref = O.coreset_streaming(h, ind, len(us), randomize=True, uniforms=us)
    assert _run(eng, h, ind, len(us), randomize=True, uniforms=us, variant=0, time_steps=True) == ref
    assert _variant(eng) == variant


def test_d2_query_beyond_the_sampling_stage_is_rejected(eng):
    """1 100 000 positions = 14 620 leaves: more than the per-step sampler's shared-memory plan holds
    (2 K nodes x 10 B <= opt-in shared memory - 16 KB).  A clean AlqError before any kernel runs."""
    rng = np.random.default_rng(11)
    full = 1100000
    h, ind, us = _d2_case(eng, rng, full, b=4)
    assert len(O.pairwise_leaves(full)) == 14620
    _raises_then_usable(eng, lambda: _run(eng, h, ind, len(us), randomize=True, uniforms=us, variant=0),
                        "partition too long for the sampling stage")


def _batched(eng, feats, inds, budgets, randomize, us=None, first=None, variant=0):
    """One batched launch over partitions p (rows feats[p], labeled indicator inds[p]); picks per partition as
    positions of its own full array.  first[p]: a full-array position that is centre 0 (or None)."""
    X, mind, vpos, cands, fp = [], [], [], [], []
    row = 0
    for p, (f, ind) in enumerate(zip(feats, inds)):
        cand, lab = np.flatnonzero(~ind), np.flatnonzero(ind)
        Xp = f[cand].cuda()
        m = torch.full((len(cand),), float("inf"), device="cuda")
        if len(lab):
            Y = f[lab].cuda()
            eng.min_dist(Xp, eng.row_norm2(Xp), Y, eng.row_norm2(Y), out=m)
        X.append(Xp)
        mind.append(m)
        vpos.append(cand)
        cands.append(cand)
        fp.append(-1 if first is None or first[p] is None else row + int(np.flatnonzero(cand == first[p])[0]))
        row += len(cand)
    off = np.concatenate(([0], np.cumsum([len(cd) for cd in cands]))).astype(np.int32)
    Xall = torch.cat(X)
    picks, _ = eng.greedy_select(Xall, eng.row_norm2(Xall), torch.cat(mind), off, budgets,
                                 uniforms=np.concatenate(us) if randomize else None,
                                 vpos=torch.as_tensor(np.concatenate(vpos).astype(np.int32)).cuda() if randomize else None,
                                 full_n=[len(ind) for ind in inds] if randomize else None,
                                 first_pick=fp, variant=variant, time_steps=True)
    out, at = [], 0
    for p, b in enumerate(budgets):
        out.append(cands[p][picks[at:at + b] - off[p]].tolist())
        at += b
    return out


def _oracle(f, ind, b, randomize, us, first=None):
    """The oracle's picks for one partition; a caller-chosen centre 0 is labeled first and uses no uniform."""
    if first is None:
        return O.coreset_streaming(f, ind, b, randomize=randomize, uniforms=us)
    ind = ind.copy()
    ind[first] = True
    return [first] + O.coreset_streaming(f, ind, b - 1, randomize=randomize, uniforms=us[1:])


@pytest.mark.parametrize("extra,variant", [(1, 2), (0, 3)])
def test_more_active_partitions_than_sms(eng, sms, extra, variant):
    """P = G + 1 active partitions cannot have one CTA each: per-step kernels.  P = G: the persistent loop."""
    rng = np.random.default_rng(400 + extra)
    P = sms + extra
    sizes = rng.integers(40, 201, P)
    feats, inds, budgets = [], [], []
    for s in sizes:
        h, _, ind = _fixture(rng, int(s), 6, 16)
        feats.append(h)
        inds.append(ind)
        budgets.append(int(rng.integers(1, 6)))
    for randomize in (False, True):
        us = [rng.random(b) for b in budgets]
        if variant == 2:
            _raises_then_usable(eng, lambda: _batched(eng, feats, inds, budgets, randomize, us, variant=3),
                                "persistent loop does not fit")
        got = _batched(eng, feats, inds, budgets, randomize, us, variant=0)
        assert _variant(eng) == variant
        for p in range(P):
            assert got[p] == _oracle(feats[p], inds[p], budgets[p], randomize, us[p]), (randomize, p)


def test_arg_max_segment_beyond_the_16_bit_row_offset(eng, sms):
    """P = G partitions, one CTA each; partition 0's CTA holds 70 000 rows, beyond the 16-bit row offset of the
    persistent arg-max word: per-step kernels."""
    rng = np.random.default_rng(500)
    sizes = [70000] + [8] * (sms - 1)
    feats, inds = [], []
    for s in sizes:
        h, _, ind = _fixture(rng, s, 3, 16)
        feats.append(h)
        inds.append(ind)
    budgets = [40] + [int(rng.integers(1, 9)) for _ in range(sms - 1)]
    assert len(sizes) == sms and sizes[0] > KEY_ROW_OFFSET
    _raises_then_usable(eng, lambda: _batched(eng, feats, inds, budgets, False, variant=3), "persistent loop does not fit")
    got = _batched(eng, feats, inds, budgets, False, variant=0)
    assert _variant(eng) == 2
    for p in range(sms):
        assert got[p] == _oracle(feats[p], inds[p], budgets[p], False, None), p


def test_row_too_large_for_the_ring(eng):
    """d = 20 480 (80 KB rows): no 3-stage ring fits, so variant=0 runs the direct-load kernel (variant 1) and
    variants 2 and 3 are refused.  The K3 contraction before it runs on tensor cores, one 20 MB row block per round.
    d = 60 000 does not fit shared memory at all."""
    rng = np.random.default_rng(600)
    n, l0, b, d = 2500, 300, 20, 20480
    h, _, ind = _fixture(rng, n, l0, d)
    us = rng.random(b)
    for randomize in (False, True):
        for forced in (3, 2):
            _raises_then_usable(eng, lambda: _run(eng, h, ind, b, randomize=randomize, uniforms=us, variant=forced),
                                "persistent loop does not fit" if forced == 3 else "variant 2 does not fit")
        ref = O.coreset_streaming(h, ind, b, randomize=randomize, uniforms=us)
        assert _run(eng, h, ind, b, randomize=randomize, uniforms=us, variant=0, time_steps=True) == ref
        assert _variant(eng) == 1
    x = torch.ones(8, 60000, device="cuda")
    mind = torch.arange(8, dtype=torch.float32, device="cuda")
    _raises_then_usable(eng, lambda: eng.greedy_select(x, eng.row_norm2(x), mind, [0, 8], [2], variant=0),
                        "row does not fit shared memory")
