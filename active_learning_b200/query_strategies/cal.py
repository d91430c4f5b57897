"""CAL, Contrastive Active Learning (Margatina, Vernikos, Barrault & Aletras, "Active Learning by Acquiring Contrastive
Examples", EMNLP 2021) on the device (kernels K18, K19, K1b).

The pool's labeled rows are the references R, its available rows the candidates.  One pool forward of the task network
gives the logits and the embeddings together (BADGE's forward; the embedding cache applies under --freeze_feature).  Each
candidate's k = min(NUM_NEIGHBORS, |R|) nearest references by the exact fp64 squared distance of the raw embeddings (K18)
score it by the mean KL divergence of their predicted distributions from the candidate's (K19), and the budget's largest
scores are taken, the lowest position on ties (K1b on the key -fl32(score)).  The spec is tests/cal_oracle.py.

CAL is undefined without labeled rows: the query raises ValueError then.  It always returns the whole budget, so it draws
nothing from NumPy beyond the pool's two shuffles.
"""
from __future__ import annotations

import numpy as np
import torch

from .coreset import PoolQuery


class CALQuery(PoolQuery):
    """The candidates whose predictions differ most from those of their nearest labeled neighbours."""
    NUM_NEIGHBORS = 10

    def _positions(self, union, is_lab, avail, budget):
        lab_pos, cand_pos = np.flatnonzero(is_lab), np.flatnonzero(avail)
        if not len(lab_pos):
            raise ValueError("CALSampler needs labeled rows: the contrastive score compares each candidate with its "
                             "labeled neighbours")
        eng = self.get_engine()
        self.feature_net.eval()
        logits, emb = self._forward_pool(union.tolist(), self.net, want_features=True)
        dev = emb.device
        lab_t = torch.as_tensor(lab_pos, device=dev)
        cand_t = torch.as_tensor(cand_pos, device=dev)
        k = min(int(self.NUM_NEIGHBORS), len(lab_pos))
        idx, _, _ = eng.knn(emb.index_select(0, cand_t), emb.index_select(0, lab_t), k)
        _, key = eng.cal_scores(logits.index_select(0, cand_t), logits.index_select(0, lab_t), idx)
        picks = eng.select_smallest(key, budget).cpu().numpy().astype(np.int64)
        return cand_pos[picks]
