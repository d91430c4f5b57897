"""BAIT (Ash, Goel, Krishnamurthy & Kakade, "Gone Fishing: Neural Active Learning with Fisher Embeddings", NeurIPS 2021) on
the device (kernels K24, K25, K26).

One pool forward of the task network gives the logits and the embeddings together (BADGE's, CAL's and ALFA-Mix's
forward; the embedding cache applies under --freeze_feature).  A row's Fisher embedding is V_x = R_x (x) h_x^T with
R_x = diag(sqrt p_x)(I - 1 p_x^T), p_x the softmax of its logits and h_x its raw embedding.  F is the pool's mean Fisher
(K24).  BAIT greedily picks the candidates that minimise tr((M + sum V^T V)^-1 F), M = lamb I plus the labeled rows'
Fisher: T = min(2 budget, #candidates) forward picks, each the largest trace decrease, then T - budget backward removals,
each the smallest increase (K26).  The inverse is kept as a dense (C D) x (C D) matrix A and every pick is a rank-C
Woodbury update of it; the per-row C x C forms h^T A_ab h and h^T (A F A)_ab h are updated with it, so a step costs
O((C D)^2 C + n D C^2) instead of recomputing every candidate's C x (C D) product.  The spec is tests/bait_oracle.py.

The dense matrices take 24 (C D)^2 bytes (0.63 GB at C = 10, D = 512 and 10 GB at D = 2048; ImageNet's C = 1000 at
D = 2048 would need 100 TB): the query checks this against the free device memory before anything is allocated
(Engine.bait_guard) and releases it before returning.  K26 holds C <= 16.  BAIT always returns the whole budget, so it draws nothing from
NumPy beyond the pool's two shuffles.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from .coreset import PoolQuery


def bait_lamb(lamb):
    """The sampler kwarg `lamb` (the ridge on the labeled Fisher, the authors' name; default 1.0) as a float: ValueError
    unless it is finite and > 0."""
    try:
        v = float(lamb)
    except (TypeError, ValueError):
        raise ValueError(f"BAITSampler: lamb={lamb!r} is not a number") from None
    if not (math.isfinite(v) and v > 0):
        raise ValueError(f"BAITSampler: lamb must be finite and > 0, got {lamb!r}")
    return v


class BAITQuery(PoolQuery):
    """Forward-backward greedy selection on the last layer's Fisher information."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.lamb = bait_lamb(kwargs.get("lamb", 1.0))

    def _positions(self, union, is_lab, avail, budget):
        eng = self.get_engine()
        self.feature_net.eval()
        logits, emb = self._forward_pool(union.tolist(), self.net, want_features=True)
        eng.bait_guard(emb.shape[0], logits.shape[1], emb.shape[1])
        try:
            p, F = eng.bait_fisher(logits, emb)
            state = eng.bait_init(emb, F, self.lamb)
            picks, _order, _fwd, _bwd = eng.bait_select(emb, p, F, state, np.flatnonzero(is_lab), np.flatnonzero(avail), budget)
        finally:
            p = F = state = None
            torch.cuda.empty_cache()
        return picks
