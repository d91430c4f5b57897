"""VAAL acquisition on the device (kernels K9 + K1b): the query of vaal_sampler.py:39-70 of
active_learning/src/query_strategies (https://arxiv.org/abs/1904.00370).

The reference runs the whole VAE on every loader batch -- encoder, reparameterize and decoder -- keeps only mu, scores
it with the discriminator and sorts the pool on the host.  Here each batch is cropped on the host before it is staged
(a 64 x 64 crop of a 224 x 224 image is 12.25x fewer bytes over PCIe), only `fc_mu(encoder(x))` runs, mu lands in a
device slab, K9 scores the slab on the tensor cores and K1b returns the `budget` smallest p, ties by pool position.
The RNG streams are left exactly as the reference leaves them: NumPy is reseeded with the VAE's crop seed per batch
(vae.py's crop index), and the torch CPU generator replays the `torch.randn(b, z)` that reparameterize draws per batch.
"""
from __future__ import annotations

import numpy as np
import torch

from .strategy import EngineMixin

CROP_H = CROP_W = 64     # vae.py:6-7


def crop_window(crop_seed, h, w):
    """vae.py's _gen_random_crop_index: (h_start, h_end, w_start, w_end) of the crop of an h x w image.  Reseeds
    NumPy's global RNG with crop_seed and draws w_start, then h_start, when both sides are >= 64; takes 0:64 (the
    whole image) when both are smaller; ValueError otherwise."""
    np.random.seed(crop_seed)
    if w < CROP_W and h < CROP_H:
        return 0, CROP_H, 0, CROP_W
    if w >= CROP_W and h >= CROP_H:
        w0 = np.random.randint(w - CROP_W + 1)
        h0 = np.random.randint(h - CROP_H + 1)
        return h0, h0 + CROP_H, w0, w0 + CROP_W
    raise ValueError("Unimplemented architecture for current image size.")


class VAALQuery(EngineMixin):
    """vaal_sampler.py: the `budget` pool rows the discriminator finds least likely to be labeled (smallest p)."""

    # the encoder ends in a view of NCHW memory (vae.py's View): batches and weights stay in the default layout
    channels_last = False

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        # trained modules: kwargs of the standalone sampler, or what the reference's own VAALSampler built and trained
        self.vae = kwargs.get("vae", getattr(self, "vae", None))
        self.discriminator = kwargs.get("discriminator", getattr(self, "discriminator", None))

    def query(self, budget):
        vae, disc = self.vae, self.discriminator
        if vae is None or disc is None:
            raise ValueError("VAALSampler.query needs the trained VAE and discriminator: pass vae= and discriminator= "
                             "(the reference's VAE / Discriminator modules, trained), or bind the query onto the "
                             "reference's VAALSampler with make_drop_in(Strategy, vaal_base=VAALSampler), whose "
                             "training loop trains them")
        if not hasattr(vae, "crop_seed"):
            raise ValueError("the VAE has no crop seed: its training loop sets one (vae.set_crop_seed) every batch")
        idxs_for_query = self.available_query_idxs()
        budget = int(min(len(idxs_for_query), budget))
        self.net.eval()
        vae.eval()
        disc.eval()
        if budget <= 0:
            return [], 0
        n = len(idxs_for_query)
        group = getattr(self, "_shard_group", None)
        sharded = group is not None and group.world_size > 1
        lo, hi = group.row_range(n) if sharded else (0, n)
        eng = self.get_engine()
        mu = self._pool_mu(idxs_for_query, lo, hi, vae)
        p = eng.vaal_scores(mu, disc)
        if sharded:
            pos_loc = eng.select_smallest(p, min(budget, hi - lo))
            pos = group.merge_smallest(p, pos_loc, lo, budget, eng, rendezvous=True)
        else:
            pos = eng.select_smallest(p, budget).cpu().numpy()
        return np.asarray(idxs_for_query, dtype=np.int64)[np.asarray(pos, dtype=np.int64)], budget

    def _pool_mu(self, idxs, lo, hi, vae):
        """mu [hi - lo, z padded to 4] of pool rows [lo, hi) on the query device.  NumPy's and torch's CPU RNG end in
        the state the reference's single-process loop over ALL rows leaves them in, whatever [lo, hi) is."""
        dev = self._query_device()
        n, z = len(idxs), vae.fc_mu.out_features
        bs = int(self.train_args["loader_te_args"]["batch_size"])
        draws = [min(bs, n - s) for s in range(0, n, bs)]    # reparameterize's torch.randn(b, z), one per batch
        seed, seen = vae.crop_seed, []

        def cropped(loader):
            for x, y, i in loader:
                hs, he, ws, we = crop_window(seed, x.shape[2], x.shape[3])
                seen.append(x.shape)
                yield x[:, :, hs:he, ws:we], y, i

        vae.to(dev)
        mu = torch.zeros((hi - lo, (z + 3) & ~3), dtype=torch.float32, device=dev)
        off = k = 0
        with torch.no_grad():
            for x, _y, _i in self._device_batches(cropped(self._loader(idxs[lo:hi])), dev):
                m = vae.fc_mu(vae.encoder(x))
                if m.shape[0] != x.shape[0]:
                    raise ValueError(f"the VAE's encoder maps {x.shape[0]} crops of {tuple(x.shape[1:])} to {m.shape[0]} "
                                     "rows: its latent_scale does not match the image size")
                if k < len(draws):
                    torch.randn(draws[k], z)     # runs on the host while the encoder runs on the device
                    k += 1
                mu[off:off + m.shape[0], :z] = m
                off += m.shape[0]
        for b in draws[k:]:
            torch.randn(b, z)
        if not seen:
            # an empty shard: the last batch of the pool still reseeded NumPy and drew its crop
            x0 = self.al_set[int(idxs[0])][0]
            crop_window(seed, x0.shape[-2], x0.shape[-1])
        return mu
