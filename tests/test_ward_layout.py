"""The Ward query's choice of distance layout (no GPU): the n x n matrix whenever it fits the free device memory, else
scipy's condensed vector, else an error naming n and both byte counts; and the row count of a condensed vector."""
import pytest

from active_learning_b200._lib import AlqError
from active_learning_b200.engine import Engine

GiB = 1 << 30
SQ, CD = Engine.ward_bytes, Engine.ward_condensed_bytes


def test_byte_counts():
    assert SQ(80000) == 8 * 80000 ** 2 + GiB                       # unchanged meaning
    assert CD(80000) == 4 * 80000 * 79999 + GiB
    assert CD(115846) == 4 * 115846 * 115845 + GiB                 # 53.7 GB + headroom


@pytest.mark.parametrize("n, free, want", [
    (2, 2 * GiB, "square"),
    (80000, 80 * 10 ** 9, "square"),                  # the reference's subset_unlabeled on an idle 80 GB card
    (80000, 40 * 10 ** 9, "condensed"),               # ... with about 40 GB taken by something else
    (80000, 20 * 10 ** 9, None),
    (104262, 85 * 10 ** 9, "condensed"),              # ImageNet-LT's available rows at 10 % labeled
    (115846, 85 * 10 ** 9, "condensed"),              # the whole ImageNet-LT train set
    (140000, 85 * 10 ** 9, "condensed"),              # about the limit of an 80 GB card
    (150000, 85 * 10 ** 9, None),
    (200000, 85 * 10 ** 9, None),
    (46500, SQ(46500), "square"),                     # the boundaries are inclusive
    (46500, SQ(46500) - 1, "condensed"),
    (46500, CD(46500), "condensed"),
    (46500, CD(46500) - 1, None),
])
def test_layout_choice(n, free, want):
    if want is None:
        with pytest.raises(AlqError, match=f"n={n} ") as e:
            Engine.ward_layout(n, free)
        assert str(SQ(n)) in str(e.value) and str(CD(n)) in str(e.value) and str(free) in str(e.value)
    else:
        assert Engine.ward_layout(n, free) == want


@pytest.mark.parametrize("n", [2, 3, 4, 1000, 65537, 92683, 115846, 4194240])
def test_condensed_rows_inverts_the_length(n):
    assert Engine.condensed_rows(n * (n - 1) // 2) == n


@pytest.mark.parametrize("length", [0, 2, 4, 11, 434, 436, 115846 * 115845 // 2 + 1, -1])
def test_condensed_rows_rejects_other_lengths(length):
    with pytest.raises(AlqError):
        Engine.condensed_rows(length)
