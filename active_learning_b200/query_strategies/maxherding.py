"""MaxHerding (Bae, Noh & Sutherland, "Generalized Coverage for More Robust Low-Budget Active Learning", ECCV 2024) on the
device (kernels K22, K23).

The pool's embeddings are L2-normalised as ProbCover normalises them, and K22 forms the Gaussian kernel matrix
K_ij = fl32(exp(-(s_ij / q))) of the exact fp64 squared distances s_ij (K7's pair arithmetic), q = 2 sigma^2.  The greedy
(K23) then maximises the generalised coverage F(S) = sum_i max_{s in L u S} K_is over the labeled rows L and the picks S,
one available row at a time: the lowest position of the largest gain.  The gains are kept incrementally: a pick changes
only the rows it now covers best, so a step reads those rows of K instead of all of it.  Once every gain is 0 (a kernel
that underflowed at a small sigma) the lowest free position is taken, so the greedy always fills the budget and there is
no NumPy draw after the two shuffles.

The n x n fp32 matrix (4 n^2 bytes: 53.7 GB at ImageNet-LT's 115 846 rows) is checked against the free device memory
before anything is allocated, and released before the query returns: nothing is kept across rounds.
"""
from __future__ import annotations

import math
import sys

import numpy as np
import torch

from .coreset import PoolQuery


def herding_q(sigma):
    """q = 2 sigma^2 (fp64) from the sampler kwarg `sigma`: required, finite and > 0, and q a finite positive normal
    number (otherwise s_ii / q can be 0 / 0)."""
    if sigma is None:
        raise ValueError("MaxHerdingSampler needs the sampler kwarg sigma (the Gaussian kernel's width, finite and > 0)")
    sigma = float(sigma)
    if not (math.isfinite(sigma) and sigma > 0):
        raise ValueError(f"MaxHerdingSampler: sigma must be finite and > 0, got {sigma}")
    q = 2.0 * sigma * sigma
    if not (math.isfinite(q) and q >= sys.float_info.min):
        raise ValueError(f"MaxHerdingSampler: 2 sigma^2 = {q} for sigma = {sigma} is not a finite positive normal number")
    return q


class MaxHerdingQuery(PoolQuery):
    """Greedy maximum generalised coverage of CoreSet's pool under a Gaussian kernel."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.sigma = kwargs.get("sigma")
        herding_q(self.sigma)

    def _positions(self, union, is_lab, avail, budget):
        eng = self.get_engine()
        feats, _ = self._features(union.tolist())
        eng.herding_guard(feats.shape[0], feats.shape[1])
        K = eng.herding_kernel(eng.normalize(feats), self.sigma)
        try:
            dev = K.device
            lab = torch.from_numpy(is_lab.astype(np.uint8)).to(dev)
            av = torch.from_numpy(avail.astype(np.uint8)).to(dev)
            picks, _m, _sum_s = eng.herding_select(K, lab, av, budget)
        finally:
            del K
            eng.herding_release()
        return picks
