"""The sharded uncertainty tail (alq_uncertainty_tail_sharded) in a group of one rank, on one GPU.  The peer-memory window
is then this GPU's own memory, but the fused launch runs select_epilogue_mgpu with the same stores, waits, fences and
tags as on a real group, and the launches that do not fuse run the top-B window exchange (alq_topb_exchange).  Inputs
are those of the fused-tail tests of test_gpu_scores.py; the result must equal the two separate kernels bit for bit,
with positions shifted by the shard's row offset."""
import pytest
import torch

from helpers import FUSED_TAIL_SHAPES, fused_tail_logits, fuses, one_rank_engine, skewed_tail_pools, tied_tail_pools

pytestmark = pytest.mark.gpu

ROW_LO_BIG = (1 << 30) + 7      # global positions stay below 2^31 for every pool here


@pytest.fixture(scope="module")
def eng(tmp_path_factory):
    with one_rank_engine(tmp_path_factory.mktemp("one_rank_group")) as e:
        yield e


def check_one_rank(eng, logits, mode, b):
    from active_learning_b200._lib import AlqError
    n, c = logits.shape
    ref_s = eng.score_softmax(logits, mode)
    ref_p = eng.select_smallest(ref_s, b)
    fused = fuses(n, c)
    for row_lo in (0, ROW_LO_BIG):
        s, p = eng.uncertainty_tail_sharded(logits, mode, b, row_lo, n, n)
        assert torch.equal(s, ref_s)
        assert torch.equal(p, ref_p + row_lo), (n, c, b, mode, row_lo)
        torch.cuda.synchronize()            # the exchange's status word is final once the stream has finished
        eng.comm_check()
        if fused:
            eng.uncertainty_tail_timing()
        else:                               # the separate kernels and alq_topb_exchange at world 1
            with pytest.raises(AlqError):
                eng.uncertainty_tail_timing()


@pytest.mark.parametrize("n,c,b", FUSED_TAIL_SHAPES)
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_one_rank_tail_equals_score_then_select(eng, n, c, b, mode):
    logits = fused_tail_logits(n, c, b, mode)
    try:
        for buckets in (1, 0):
            eng.set_option("tail_buckets", buckets)
            check_one_rank(eng, logits, mode, b)
    finally:
        eng.set_option("tail_buckets", 1)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_one_rank_tail_with_skewed_scores(eng, mode):
    for logits, b in skewed_tail_pools(mode):
        check_one_rank(eng, logits, mode, b)


def test_one_rank_tail_with_massive_ties(eng):
    for logits, b in tied_tail_pools():
        for mode in (0, 1, 2):
            check_one_rank(eng, logits, mode, b)
    check_one_rank(eng, torch.zeros(70000, 16, device="cuda"), 0, 5000)
