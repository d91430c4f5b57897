"""What the exactness claims of the tensor-core kernels rest on, read from their sources.

test_gpu_tf32_bound.py measures the 3xTF32 bound through K3 and DESIGN section 4 applies it to K9, K13, K15 and K18,
because all five issue one chain, alq_wgmma.cuh's tc::ring_mma, and take the band's coefficient from one place,
tc::band_coef.  The distances they certify are K7's pair arithmetic, written once in alq_common.cuh (d2_step, exact_d2),
and the ring is correct only while its producer and consumers walk one k-block sequence, which K9, K15 and K18 take
from tc::ring_produce_rows and tc::ring_tile."""
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "active_learning_b200", "csrc")
RING_KERNELS = {"alq_mindist_tc.cu": "K3", "alq_vaal.cu": "K9", "alq_probcover.cu": "K13", "alq_typiclust.cu": "K15",
                "alq_cal.cu": "K18"}


def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _all_sources():
    return {name: _src(name) for name in sorted(os.listdir(CSRC)) if name.endswith((".cu", ".cuh"))}


def test_the_ring_kernels_issue_only_the_rings_chain():
    """None of the five may issue MMAs, TMA loads or barriers of its own; K3 calls ring_mma, the others ring_tile."""
    for name, k in RING_KERNELS.items():
        src = _src(name)
        assert ("ring_mma(" if k == "K3" else "ring_tile(") in src, (k, name)
        for own in ("wgmma_tf32(", "tma_load_2d(", "mbar_init("):
            assert own not in src, (k, name, own)
    assert "ring_mma(" in _src("alq_wgmma.cuh").split("void ring_tile(")[1].split("\n}\n")[0]


def test_the_row_block_kernels_share_one_producer():
    for name in ("alq_vaal.cu", "alq_typiclust.cu", "alq_cal.cu"):
        src = _src(name)
        assert "ring_produce_rows(" in src, name
        assert "ring_load(" not in src, name


def test_the_exact_pair_arithmetic_and_the_band_coefficient_are_written_once():
    srcs = _all_sources()
    assert [n for n, s in srcs.items() if "__dmul_rn(df, df)" in s] == ["alq_common.cuh"]
    assert [n for n, s in srcs.items() if "ldexp(1.0, -20)" in s] == ["alq_wgmma.cuh"]
    for name in ("alq_probcover.cu", "alq_typiclust.cu", "alq_cal.cu"):
        assert "tc::band_coef(d)" in srcs[name], name


def test_every_scratch_layout_is_written_once():
    """Each entry point's takes both size and carve its scratch (alq_scratch_carve): no list of sizes beside them, no
    cursor or reservation outside the helper, and the arena's growth rule in alq_ctx.cu alone."""
    srcs = _all_sources()
    assert [n for n, s in srcs.items() if "scratch_" "need" in s] == []      # a size list beside the takes
    assert [n for n, s in srcs.items() if re.search(r"\bScratchCursor\s*(\w+\s*)?[({]", s)] == ["alq_common.cuh"]
    for fn in ("alq_scratch_reserve", "alq_arena2_reserve"):
        calls = {n: len(re.findall(r"\b%s\(" % fn, s)) for n, s in srcs.items()}
        # alq_common.cuh: the declaration and the helper's call; alq_ctx.cu: the definition
        assert {n: k for n, k in calls.items() if k} == {"alq_common.cuh": 2, "alq_ctx.cu": 1}, fn
    assert [n for n, s in srcs.items() if re.search(r"\(\s*\w+\s*>>\s*2\s*\)\s*\+\s*\(\s*1u?\s*<<\s*20\s*\)", s)] == ["alq_ctx.cu"]
