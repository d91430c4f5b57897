"""The twin of BASE's parallel route (tests/base_route_twin.py) against the oracle's class loop, and each key
constructor against the branch it is built for."""
import numpy as np
import pytest
import torch

import base_route_twin as T
from oracle import al_oracle as O


def oracle_picks(K, budget, seed=0):
    mm, radius, pred = T.split_keys(K, seed)
    return O.base_select(torch.from_numpy(mm), torch.from_numpy(radius), torch.from_numpy(pred).long(), budget, K.shape[1])


def check(K, budget):
    picks, fallbacks, fail, dup = T.twin_select(K, budget)
    assert dup == 0
    assert picks.tolist() == oracle_picks(K, budget).tolist()
    return fallbacks, fail


def test_split_keys_gives_the_oracle_the_key_matrix():
    K = T.random_keys(300, 7, 1)
    mm, radius, pred = T.split_keys(K, 3)
    for c in range(7):
        key = torch.where(torch.from_numpy(pred).long() == c, torch.from_numpy(mm), torch.from_numpy(radius)[:, c])
        assert np.array_equal(key.numpy(), K[:, c])


def test_pack_orders_like_a_stable_sort():
    key = np.array([0.5, -0.0, 0.0, -1.0, np.inf, 0.5, -np.inf, 1e-30], dtype=np.float32)
    assert np.argsort(T.pack(key)).tolist() == np.argsort(key, kind="stable").tolist()
    assert T.ord32(np.float32(-0.0)) == T.ord32(np.float32(0.0)) and int(T.ord32(np.float32(np.inf))) == T.ORD_INF


@pytest.mark.parametrize("n,c,budget,quantise", [(3000, 20, 300, False), (5000, 40, 400, True), (2000, 16, 16 * 32, False),
                                                 (900, 24, 23, False), (1234, 17, 200, True), (4097, 3, 90, False)])
def test_twin_matches_oracle_on_random_keys(n, c, budget, quantise):
    fallbacks, fail = check(T.random_keys(n, c, n + c, quantise), budget)
    assert not fail.any() and fallbacks == []


@pytest.mark.parametrize("c,targets", [(20, [0, 7, 19]), (1003, [0, 500, 1001, 1002])])
def test_forced_fail_sets_exactly_the_targeted_flags(c, targets):
    n = 4500 if c > 100 else 6000
    budget = c * 3
    K = T.forced_fail(n, c, targets, 5)
    fallbacks, fail = check(K, budget)
    assert np.flatnonzero(fail).tolist() == targets
    assert fallbacks == targets


def test_forced_fail_without_the_dropped_pair_check_is_wrong():
    """The planted class is exactly where a list built from the kept pairs alone differs from the true top list."""
    K = T.forced_fail(6000, 20, [7], 5)
    lst, bad = T.class_candidates(K[:, 7], 15)
    truth = np.sort(T.pack(K[:, 7]))[:T.list_len(15)]
    assert bad and not np.array_equal(lst[:T.list_len(15)], truth)
    assert np.array_equal(T.class_candidates(K[:, 6], 15)[0][:T.list_len(15)], np.sort(T.pack(K[:, 6]))[:T.list_len(15)])


def test_exhausted_lists_fall_back_class_after_class():
    """cnt = 10, len = 42: classes 0-3 take 40 rows of the shared column, class 4 sees 2 free entries, every later
    list is entirely taken."""
    c, budget = 100, 1000
    fallbacks, fail = check(T.exhausted(20000, c, 2), budget)
    assert not fail.any()
    assert fallbacks == list(range(4, c))


def test_exhausted_only_at_the_last_class():
    c, cnt = 20, 10
    fallbacks, fail = check(T.exhausted_at(5000, c, cnt, 4), c * cnt)
    assert fallbacks == [c - 1] and not fail[c - 1]


def test_ties_and_infinite_keys():
    c, budget = 30, 300
    K = T.ties(8000, c, 6, short_class=0, short_finite=4)
    fallbacks, fail = check(K, budget)
    assert fallbacks[0] == 0        # 4 finite keys, 10 picks: the list runs out of finite rows, the step takes 6 at +inf
    assert len(fallbacks) > 1       # the runs of zeros at low rows are shared: later lists run out of free rows
    ln = T.list_len(10)
    truth = np.sort(T.pack(K[:, 1])) >> np.uint64(32)
    assert truth[0] == truth[ln - 1] == truth[ln] == truth[1000]        # the list's last entry inside a run of ties
    assert np.isinf(K[:800, 3]).all() and np.isfinite(K[800:, 3]).all()


def test_budget_below_the_class_count():
    c, budget = 40, 25
    K = T.forced_fail(5000, c, [3, 30], 8)
    fallbacks, fail = check(K, budget)
    assert fallbacks == [3]                                 # class 30 takes no row, its flag is never consulted
    assert T.counts(budget, c)[30] == 0


def test_double_selection_is_reported():
    K = np.full((64, 16), np.inf, dtype=np.float32)
    picks, fallbacks, fail, dup = T.twin_select(K, 40)
    assert fallbacks == list(range(16)) and dup > 0
    with pytest.raises(AssertionError):
        oracle_picks(K, 40)


def test_launch_delta_counts_the_resumes():
    sel = {1: 1, 10: 1, 11: 1}
    assert T.launch_delta([], 20, 200, sel) == 2
    assert T.launch_delta([19], 20, 200, sel) == 2 + 3                # the walk ends with the fallback: no resume
    assert T.launch_delta([3, 19], 20, 200, sel) == 2 + 4 + 3
    assert T.sequential_delta(20, 205, sel) == 20 * 3
    assert T.sequential_delta(40, 25, sel) == 25 * 3
