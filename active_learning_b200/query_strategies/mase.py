"""MASE / BASE acquisition on the device (kernel K6 + K1b): SURVEY.md section 8f rank 2.

Query skeletons of active_learning/src/query_strategies/mase_sampler.py:19-27 and base_sampler.py:12-44.  The
reference broadcasts (B, C, M) tensors per loader batch to measure how far every embedding is from each pairwise
decision boundary of the linear head; with the algebra carried out that distance is the logit gap over the head
geometry, |z_p - z_c| / |w_p - w_c| (include/alq.h, K6), so the tail is one C x C table per query and one streaming
pass over the logits slab the forward already produced.  Selection (one stable sort for MASE, one per class for
BASE) stays on the device; only `budget` int32 positions return to the host.
"""
from __future__ import annotations

import numpy as np
import torch

from .._lib import AlqError
from .strategy import EngineMixin


class MASEQuery(EngineMixin):
    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.cache_embeddings = kwargs.get("cache_embeddings", True)
        self.channels_last = kwargs.get("channels_last", True)
        self.mase_self_check = kwargs.get("mase_self_check", True)

    # ---- mase_sampler.py:19-27 ---------------------------------------------------------------------
    def query(self, budget):
        idxs_for_query = self.available_query_idxs(boolean=False, shuffle=False)
        budget = int(min(len(idxs_for_query), budget))
        if budget <= 0:
            return [], 0
        eng = self.get_engine()
        group = getattr(self, "_shard_group", None)
        if group is not None and group.world_size > 1:
            lo, hi = group.row_range(len(idxs_for_query))
            min_margins, _, _ = self._margins_device(idxs_for_query[lo:hi], want_per_class=False)
            pos_loc = eng.select_smallest(min_margins, min(budget, hi - lo))
            pos = group.merge_smallest(min_margins, pos_loc, lo, budget, eng, rendezvous=True)
        else:
            min_margins, _, _ = self._margins_device(idxs_for_query, want_per_class=False)
            pos = eng.select_smallest(min_margins, budget).cpu().numpy()
        labeled_idxs = np.asarray(idxs_for_query)[pos].tolist()
        return labeled_idxs, budget

    # ---- mase_sampler.py:29-102 (the head through EngineMixin._head, :46-49) ---------------------------
    def _margins_device(self, idxs, want_per_class, dataset=None, labels_out=None):
        """(min_margins [n] fp32, pred [n] int32, per_class [n, C] fp32 or None), all on the query device."""
        eng = self.get_engine()
        self.net.eval()
        logits, _ = self._forward_pool(idxs, self.net, want_features=False, dataset=dataset, labels_out=labels_out)
        weight, _bias = self._head()
        ginv = eng.class_gap_inv(weight.detach().to(logits.device, torch.float32))
        min_margins, pred, radius = eng.mase_margins(logits, ginv, want_per_class=want_per_class)
        if self.mase_self_check and len(idxs):
            self._check_last_batch(idxs, ginv, dataset)
        return min_margins, pred, radius

    def _check_last_batch(self, idxs, ginv, dataset=None):
        """The reference's "check the method works" (:88-93): move the embeddings of the last loader batch onto
        their nearest boundary and assert that the two largest logits meet there."""
        bs = int(self.train_args["loader_te_args"]["batch_size"])
        tail = len(idxs) % bs or min(bs, len(idxs))
        last = list(idxs[len(idxs) - tail:])
        with torch.no_grad():
            logits, emb = self._forward_pool(last, self.net, want_features=True, dataset=dataset)
            weight, _bias = self._head()
            m = weight.shape[1]
            emb = emb[:, :m]
            _mn, pred, radius = self.get_engine().mase_margins(logits, ginv, want_per_class=True)
            cstar = radius.min(dim=1).indices
            w = weight.detach().to(emb.device, torch.float32)
            wd = w[pred.long()] - w[cstar]
            gap = logits.gather(1, pred.long()[:, None])[:, 0] - logits.gather(1, cstar[:, None])[:, 0]
            lam = 2 * gap / (wd ** 2).sum(dim=1)
            logits_adv = self.net(emb + (-wd * lam[:, None] / 2), specify_input_layer="finalembed")
            top = torch.topk(logits_adv, k=2, dim=1, largest=True)
            assert (top.values[:, 0] - top.values[:, 1]).abs().mean() < 0.0001

    def compute_margins(self, idxs_for_query, use_training_augmentation=False):
        """API of mase_sampler.py:29: (min_margins, per_class_margins, pred_labels, true_labels) as CPU tensors."""
        labels = []
        dataset = self.train_set if use_training_augmentation else None
        mm, pred, radius = self._margins_device(idxs_for_query, want_per_class=True, dataset=dataset, labels_out=labels)
        true_labels = torch.cat(labels, dim=0) if labels else torch.empty(0, dtype=torch.int64)
        return mm.cpu(), radius.cpu(), pred.long().cpu(), true_labels


class BASEQuery(MASEQuery):
    # ---- base_sampler.py:12-44 ---------------------------------------------------------------------
    def query(self, budget):
        idxs_for_query = self.available_query_idxs(boolean=False, shuffle=False)
        budget = int(min(len(idxs_for_query), budget))
        if budget <= 0:
            return [], 0
        eng = self.get_engine()
        group = getattr(self, "_shard_group", None)
        if group is not None and group.world_size > 1:
            # rows sharded for the forward + K6; the class loop excludes rows across shards, so every rank runs it on
            # the gathered margins (N x C fp32 over NVLink once, replicated bookkeeping, identical picks)
            n = len(idxs_for_query)
            counts = [hi - lo for lo, hi in (group.row_range(n, q) for q in range(group.world_size))]
            lo, hi = group.row_range(n)
            mm, pred, radius = self._margins_device(idxs_for_query[lo:hi], want_per_class=True)
            mm, pred, radius = (group.all_gather_rows(t, counts) for t in (mm, pred, radius))
        else:
            mm, pred, radius = self._margins_device(idxs_for_query, want_per_class=True)
        try:
            pos = eng.base_select(mm, radius, pred, budget).cpu().numpy()
        except AlqError as e:
            if "selected twice" in str(e):
                raise AssertionError(str(e)) from e          # base_sampler.py:40
            raise
        labeled_idxs = np.asarray(idxs_for_query)[pos].tolist()
        return labeled_idxs, budget
