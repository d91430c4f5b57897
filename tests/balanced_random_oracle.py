"""CPU restatement of the reference's BalancedRandomSampler.query (balanced_random_sampler.py:17-101 of
active_learning/src/query_strategies), line by line with its threshold loop kept.  One deviation: the rows of a class are
taken with `.nonzero().reshape(-1)` where the reference uses `.squeeze()`, which turns a class with exactly one
available row into a 0-d tensor and raises IndexError; `torch.randperm(1)` draws nothing, so the RNG stream is the
one the reference would have reached.  tests/golden/make_golden_balanced_random.py checks it against the reference."""
import hashlib

import numpy as np
import torch


def reference_budgets(labels_available_count, budget, num_classes):
    """balanced_random_sampler.py:43-72 as written: (per-class budgets int32, thres, oneadd, argsort permutation)."""
    labels_available_count = np.asarray(labels_available_count, dtype=np.float64)
    sort_idxs = np.argsort(labels_available_count)
    labels_count_sorted = labels_available_count[sort_idxs]
    reverse_sort_idxs = np.empty_like(sort_idxs)
    reverse_sort_idxs[sort_idxs] = np.arange(len(labels_available_count))
    thres = budget // num_classes
    doneflag = False
    while doneflag is False:
        count_smallerequal = np.where(labels_count_sorted <= thres, labels_count_sorted, 0).sum()
        count_largermin = np.where(labels_count_sorted > thres, thres, 0).sum()
        for oneadd in range((labels_count_sorted > thres).sum() + 1):
            cum_count = count_smallerequal + count_largermin + oneadd
            if cum_count == budget:
                doneflag = True
                break
        if doneflag:
            break
        else:
            thres += 1
    num_classes_sample_count = np.where(labels_count_sorted <= thres, labels_count_sorted, thres)
    if oneadd > 0:
        num_classes_sample_count[-oneadd:] = thres + 1
    return num_classes_sample_count[reverse_sort_idxs].astype(np.int32), thres, oneadd, sort_idxs


def balanced_random_query(targets, idxs_for_query, num_classes, budget):
    """The reference's query on the labels `targets` and the boolean mask `idxs_for_query`
    (available_query_idxs(boolean=True)): (list of Python ints, budget)."""
    labels = torch.Tensor(targets)
    idxs_for_query = torch.Tensor(idxs_for_query).bool()
    budget = int(min(idxs_for_query.sum(), budget))

    labels_for_query = labels.numpy()[idxs_for_query]
    labels_available, labels_available_count = np.unique(labels_for_query, return_counts=True)
    labels_available_count_all = np.zeros(num_classes)
    labels_available_count_all[labels_available.astype(np.int32)] = labels_available_count
    labels_available_count = labels_available_count_all

    num_classes_sample_count = reference_budgets(labels_available_count, budget, num_classes)[0]
    assert len(num_classes_sample_count) == num_classes
    assert num_classes_sample_count.sum() == budget
    assert (num_classes_sample_count > labels_available_count).sum() == 0

    labeled_idxs = []
    for c in range(num_classes):
        cur_class_budget = num_classes_sample_count[c]
        if cur_class_budget == 0:
            continue
        cur_available_idxs = torch.where(labels == c, idxs_for_query, False)
        cur_labeled_idxs = cur_available_idxs.nonzero().reshape(-1)
        cur_labeled_idxs = cur_labeled_idxs[torch.randperm(cur_labeled_idxs.size(0))]
        cur_labeled_idxs = cur_labeled_idxs[:cur_class_budget]
        labeled_idxs += cur_labeled_idxs.tolist()

    assert np.unique(labeled_idxs).shape[0] == budget
    return labeled_idxs, budget


def torch_rng_digest():
    return hashlib.sha256(torch.get_rng_state().numpy().tobytes()).hexdigest()


def np_rng_digest():
    st = np.random.get_state()
    return hashlib.sha256(st[1].tobytes() + repr(st[2:]).encode()).hexdigest()
