"""Error behaviour of the C ABI: bad arguments become AlqError with the library's message (the reference
raises Python exceptions; there are no silent fallbacks)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from active_learning_b200.engine import Engine
    return Engine()


def test_invalid_arguments_raise(eng):
    from active_learning_b200._lib import AlqError
    x = torch.randn(64, 12, device="cuda")
    with pytest.raises(AlqError, match="CUDA tensor"):
        eng.score_softmax(torch.randn(4, 4), 0)
    with pytest.raises(AlqError, match="float32"):
        eng.score_softmax(x.double(), 0)
    with pytest.raises(AlqError, match="mode"):
        eng.score_softmax(x, 7)
    with pytest.raises(AlqError, match="b <= n"):
        eng.select_smallest(torch.rand(10, device="cuda"), 11)
    xn = eng.row_norm2(x)
    odd = torch.randn(64, 10, device="cuda")          # d % 4 != 0
    with pytest.raises(AlqError, match="multiples of 4"):
        eng.min_dist(odd, eng.row_norm2(odd), odd, eng.row_norm2(odd))
    mind = torch.zeros(64, device="cuda")
    with pytest.raises(AlqError, match="budget"):
        eng.greedy_select(x, xn, mind, [0, 64], [65])
    with pytest.raises(AlqError, match="part_off"):
        eng.greedy_select(x, xn, mind, [0, 60], [5])
    with pytest.raises(AlqError, match="vpos"):
        eng.greedy_select(x, xn, mind, [0, 64], [5], uniforms=np.zeros(5))
    with pytest.raises(AlqError, match="shard_off"):
        eng.greedy_select(x, xn, mind, [0, 64], [5], shard_off=[0, 32, 64])     # no multi-GPU group on this context
    with pytest.raises(AlqError, match="unknown option"):
        eng.set_option("no_such_knob", 1)
    # the engine is still usable after errors
    assert eng.greedy_select(x, xn, mind.fill_(float("inf")), [0, 64], [3], first_pick=[5]).tolist()[0] == 5


def test_empty_and_degenerate_inputs(eng):
    assert eng.score_softmax(torch.empty(0, 10, device="cuda"), 0).numel() == 0
    assert eng.select_smallest(torch.rand(5, device="cuda"), 0).numel() == 0
    one = torch.tensor([[1.0, 1.0, 1.0, 1.0]], device="cuda")
    assert float(eng.score_softmax(one, 0)) == 0.0                    # all logits equal: margin 0
    assert abs(float(eng.score_softmax(one, 1)) - 0.25) < 1e-7
    x = torch.zeros(8, 4, device="cuda")                             # all rows identical
    picks = eng.greedy_select(x, eng.row_norm2(x), torch.zeros(8, device="cuda"), [0, 8], [8])
    assert picks.tolist() == list(range(8))                          # every tie resolves to the lowest row


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs a second GPU")
def test_int32_and_mask_arguments_on_another_gpu_are_refused(eng):
    """Their pointers would be another device's addresses: refused before any launch, as the class and balancing calls
    refuse them."""
    from active_learning_b200._lib import AlqError
    other = torch.device("cuda", (eng.device_index + 1) % torch.cuda.device_count())
    n = 64
    x = torch.nn.functional.normalize(torch.randn(n, 8, device=eng.device), dim=1)
    mask = torch.zeros(n, dtype=torch.uint8, device=other)
    labels = torch.zeros(n, dtype=torch.int32, device=other)
    with pytest.raises(AlqError, match="herding_select: labeled"):
        eng.herding_select(torch.eye(n, device=eng.device), mask, mask.to(eng.device), 1)
    row_ptr = torch.zeros(n + 1, dtype=torch.int64, device=eng.device)
    with pytest.raises(AlqError, match="probcover_select: labeled"):
        eng.probcover_select(row_ptr, torch.zeros(0, dtype=torch.int32, device=eng.device), mask, 1)
    with pytest.raises(AlqError, match="kmeans_assign: labels"):
        eng.kmeans_assign(x, x[:4].clone(), labels)
    with pytest.raises(AlqError, match="kmeans_update: labels"):
        eng.kmeans_update(x, labels, x[:4].clone())
    with pytest.raises(AlqError, match="kmeans_nearest: labels"):
        eng.kmeans_nearest(x, labels, x[:4].clone())
