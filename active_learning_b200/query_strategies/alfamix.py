"""ALFA-Mix (Parvaneh, Abbasnejad, Teney, Haffari, van den Hengel & Shi, "Active Learning by Feature Mixing", CVPR 2022)
on the device (kernels K16, K20, K13's normalise, K5, K15, K21).

The pool is CoreSet's (`get_idxs_for_coreset`: the same two shuffles, subset_labeled / subset_unlabeled honoured); its
available rows are the candidates.  One pool forward of the task network gives the logits and the embeddings together
(BADGE's and CAL's forward; the embedding cache applies under --freeze_feature).  The anchors are the fl32 means of the
labeled embeddings per class (K16), a class with no labeled row taking the mean of all of them.

The paper mixes each candidate's embedding with every anchor, z + alpha * (a_c - z), at the closed-form alpha that steps
along the loss gradient, and marks the candidate when the head's prediction changes.  With the algebra carried out, the
mixed logits are l + t W g / |g| with t = eps |a_c - z| and g = W^T (p - e_yhat), so the whole (candidate, anchor) loop
is one number per row, rho = sqrt(D) t* / max_c |a_c - z| (K20): the row flips for some anchor at cap eps = kappa /
sqrt(D) exactly when rho < kappa.  The caps kappa_j = j * alpha_step grow until more than `budget` rows flip (or the
last, j = ceil(1 / alpha_step)).  If no more rows than the budget flip they are all taken; otherwise the flipped rows,
L2-normalised, are clustered by TypiClust's k-means into `budget` clusters and each non-empty cluster gives its row
nearest the centre (K21).  The rest of the budget is ProbCover's random fill.  The spec is tests/alfamix_oracle.py.

ALFA-Mix is undefined without labeled rows: the query raises ValueError then.  NumPy draws: the pool's two shuffles, the
k-means seeding when it runs, the fill when there is a remainder.  The head moves every round, so nothing but the
embedding cache is kept across rounds.  In a ShardGroup every rank runs the whole query on its own GPU and returns the
same picks.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from .balanced_random import _host_labels
from .coreset import CoresetQuery


def cap_walk(rho, budget, alpha_step):
    """Positions of the rows with rho < kappa_j for the first j in 1 .. ceil(1 / alpha_step) whose set holds more than
    `budget` rows (kappa_j = j * alpha_step in fp64), else for the last j.  The first such j is the smallest with
    kappa_j > the (budget + 1)-th smallest rho, found without walking the caps one by one."""
    rho = np.asarray(rho, dtype=np.float64)
    last = math.ceil(1.0 / alpha_step)
    j = last
    if len(rho) > budget:
        v = float(np.partition(rho, budget)[budget])
        if v < last * alpha_step:
            j = max(1, min(last, int(v // alpha_step)))
            while j > 1 and (j - 1) * alpha_step > v:
                j -= 1
            while j * alpha_step <= v:
                j += 1
    return np.flatnonzero(rho < j * alpha_step)


class ALFAMixQuery(CoresetQuery):
    """The rows whose prediction feature mixing with the class anchors changes, spread by k-means."""
    ALPHA_STEP = 2.0 ** -5
    MAX_ITER = 100

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        step = kwargs.get("alpha_step", self.ALPHA_STEP)
        try:
            step = float(step)
        except (TypeError, ValueError):
            raise ValueError(f"ALFAMixSampler: alpha_step={step!r} is not a number") from None
        if not (math.isfinite(step) and 0.0 < step <= 1.0):
            raise ValueError(f"ALFAMixSampler: alpha_step={step!r} must be finite and in (0, 1]")
        self.alpha_step = step

    def _anchors(self, emb_lab, labels, num_classes):
        """[C, Dp]: the fl32 mean of the labeled rows of each class (K16), the mean of all labeled rows for a class
        without one."""
        eng = self.get_engine()
        dev = emb_lab.device
        mean = torch.zeros((1, emb_lab.shape[1]), dtype=torch.float32, device=dev)
        eng.kmeans_update(emb_lab, torch.zeros(emb_lab.shape[0], dtype=torch.int32, device=dev), mean)
        anchors = mean.expand(num_classes, -1).contiguous()
        return eng.kmeans_update(emb_lab, torch.as_tensor(labels.astype(np.int32), device=dev), anchors)

    def query(self, budget):
        union = np.asarray(self.get_idxs_for_coreset(), dtype=np.int64)      # RNG: two permutations
        is_lab = self.already_labeled_idxs(boolean=True)[union]
        avail = self.available_query_idxs(boolean=True)[union]
        budget = int(min(int(avail.sum()), budget))
        if budget <= 0:
            return [], 0
        lab_pos, cand_pos = np.flatnonzero(is_lab), np.flatnonzero(avail)
        if not len(lab_pos):
            raise ValueError("ALFAMixSampler needs labeled rows: the anchors are the labeled rows' class means")
        eng = self.get_engine()
        weight, _ = self._head()
        num_classes = int(weight.shape[0])
        labels = _host_labels(self.al_set.targets)[union[lab_pos]]
        if labels.size and (labels.min() < 0 or labels.max() >= num_classes):
            raise ValueError(f"ALFAMixSampler: labeled rows carry labels outside [0, {num_classes})")
        self.feature_net.eval()
        logits, emb = self._forward_pool(union.tolist(), self.net, want_features=True)
        dev = emb.device
        cand_t = torch.as_tensor(cand_pos, device=dev)
        anchors = self._anchors(emb.index_select(0, torch.as_tensor(lab_pos, device=dev)), labels, num_classes)
        rho = eng.alfamix_rho(logits.index_select(0, cand_t), emb.index_select(0, cand_t), anchors,
                              weight.detach().to(dev, torch.float32))
        cand = cand_pos[cap_walk(rho.cpu().numpy(), budget, self.alpha_step)]
        if len(cand) <= budget:
            picks = cand
        else:
            xhat = eng.normalize(emb.index_select(0, torch.as_tensor(cand, device=dev)))
            first = int(np.random.choice(len(cand)))                          # TypiClust's seeding draws
            unif = np.random.random_sample(budget - 1)
            km_labels, centres, _, _ = eng.kmeans(xhat, first, unif, budget, self.MAX_ITER)
            near = eng.kmeans_nearest(xhat, km_labels, centres)
            picks = cand[near[near >= 0]]
        rest = budget - len(picks)
        if rest > 0:
            free = avail.copy()
            free[picks] = False
            picks = np.concatenate([picks, np.random.choice(np.flatnonzero(free), rest, replace=False)])
        labeled_idxs_cur_rd = union[picks].tolist()
        return labeled_idxs_cur_rd, len(labeled_idxs_cur_rd)
