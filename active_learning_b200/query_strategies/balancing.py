"""BalancingSampler on the device (SURVEY.md section 8f rank 4): "Active Learning for Imbalanced Datasets" (WACV 2020).

Query skeleton of active_learning/src/query_strategies/balancing_sampler.py:26-134, one pick per step.  The class
histogram test (:66-82), the RNG draw of the random branch (:124) and the mask updates (:127-128) are host bookkeeping
and stay literally the reference's (tiny torch-CPU tensors, so every promotion and division rounds the same way).
What moves to the GPU is the part that scales with the pool: the embeddings never leave the device, class centres are
kept as running per-class sums, the two distance fields of a balancing step are K3 calls (`alq_min_dist`, min against
the rarest centre and max over the majority centres) and the masked ratio arg-min is `alq_ratio_argmin`; one int32
returns to the host per step.

Rounding: the class centres here are running per-class sums divided by (count + 1e-5); the reference builds
1 / (count + 1e-5) first and multiplies inside a matmul (:86-88).  The two are equal in exact arithmetic and differ in
the last fp32 bits, so a balancing step whose two best ratios are closer than ~1e-6 relative may pick the other row
than the reference does.  The golden fixtures (tests/golden/reference_golden_balancing.npz) are pick-for-pick
identical; outside them the guarantee is "same pick unless the reference's own arg-min is decided by fp32 rounding".
"""
from __future__ import annotations

import numpy as np
import torch

from .strategy import EngineMixin


class BalancingQuery(EngineMixin):
    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.freeze_feature = kwargs["freeze_feature"]          # required, like balancing_sampler.py:24
        self._bal_cache = None

    def _pool_embeddings(self):
        """Embeddings [n_pool, D padded to x4] on the device and the pool's labels (:39-58); kept across rounds under
        --freeze_feature like the reference's saved_embeddings / saved_ys."""
        if self.freeze_feature and getattr(self, "_bal_cache", None) is not None:
            return self._bal_cache
        labels = []
        self.feature_net.eval()
        _, emb = self._forward_pool(list(range(self.n_pool)), self.feature_net, want_features=True, labels_out=labels)
        ys = torch.cat([torch.as_tensor(b).reshape(-1) for b in labels], dim=0).to(torch.int64)
        if self.freeze_feature:
            self._bal_cache = (emb, ys)
        return emb, ys

    def query(self, budget):
        self.feature_net = self.net
        idxs_for_query = self.available_query_idxs(boolean=True)
        idxs_labeled = self.already_labeled_idxs(boolean=True)
        labeled_idxs_cur_rd = []
        emb, ys = self._pool_embeddings()
        eng = self.get_engine()
        dev = emb.device
        C = self.num_classes
        budget = int(min(idxs_for_query.sum(), budget))
        if budget <= 0:
            return labeled_idxs_cur_rd, 0
        # device state: per-class embedding sums, row norms, availability mask
        ys_dev = ys.to(dev)
        lab_rows = torch.from_numpy(np.flatnonzero(idxs_labeled)).to(dev)
        sums = torch.zeros((C, emb.shape[1]), dtype=torch.float32, device=dev)
        if lab_rows.numel():
            sums.index_add_(0, ys_dev[lab_rows], emb[lab_rows])
        xn = eng.row_norm2(emb)
        avail = torch.from_numpy(idxs_for_query.astype(np.uint8)).to(dev)
        hist = torch.bincount(ys[torch.from_numpy(idxs_labeled)], minlength=C)[:C]     # labeled rows per class (int64)
        for step in range(budget):
            majority = self._needs_balancing(hist, budget - step)
            if majority is not None:
                rare_n, rare = hist.min(dim=0)                                       # first index among the rarest
                rows = torch.cat([rare.reshape(1), torch.nonzero(majority).reshape(-1)]).to(dev)
                centres = sums[rows] / (hist.to(torch.float32).to(dev)[rows] + 1e-5)[:, None]      # :86-88
                cn = eng.row_norm2(centres)
                far = eng.min_dist(emb, xn, centres[1:], cn[1:], reduce_max=True)    # largest d2 to a majority centre
                near = eng.min_dist(emb, xn, centres[:1], cn[:1]) if rare_n != 0 else None   # :104-107: numerator 1
                pick = np.int64(eng.ratio_argmin(near, far, avail))                  # :115-121
            else:
                pick = np.random.choice(np.where(idxs_for_query.squeeze() == True)[0])   # noqa: E712  :124
            idxs_for_query[pick] = False
            idxs_labeled[pick] = True
            labeled_idxs_cur_rd.append(pick)
            cls = int(ys[int(pick)])
            hist[cls] += 1
            sums[cls] += emb[int(pick)]
            avail[int(pick)] = 0
        return labeled_idxs_cur_rd, len(labeled_idxs_cur_rd)

    @staticmethod
    def _needs_balancing(hist, remaining):
        """The imbalance test of balancing_sampler.py:66-82 on the labeled-class histogram, evaluated with the same
        torch-CPU promotions (int64 counts against their fp32 mean, true division of the sums).  Returns the boolean
        mask of the majority classes if the step must balance, None if it draws at random."""
        mean = hist.float().mean()
        above, rest = hist > mean, hist <= mean
        spread = hist[above].sum() / above.sum() - hist[rest].sum() / rest.sum()     # NaN when no class is above
        return above if bool(remaining <= rest.sum() * spread) else None
