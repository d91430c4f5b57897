"""CPU restatement of the reference's VAAL query (vaal_sampler.py:39-70 of active_learning/src/query_strategies) and
modules with the state-dict layout of its VAE (vae.py) and Discriminator (vaal_discriminator.py), written from the
layer lists.  The query runs the whole VAE per loader batch -- crop, encoder, fc_mu / fc_logvar, reparameterize,
decoder -- exactly as the reference does, so it consumes the RNG streams the same way; tests/golden/make_golden_vaal.py
checks it against the reference itself, and tools/vaal_time.py times it on the GPU as the baseline arm."""
import hashlib

import numpy as np
import torch
import torch.nn as nn
from torch.utils.data import DataLoader, Subset

CROP = 64


class Reshape(nn.Module):
    def __init__(self, *shape):
        super().__init__()
        self.shape = shape

    def forward(self, x):
        return x.view(self.shape)


class VAE(nn.Module):
    """4 stride-2 4x4 convolutions (3 -> 128 -> 256 -> 512 -> 1024, each BatchNorm + ReLU, no bias), flattened to
    4096 ls^2 features; fc_mu / fc_logvar to z; the decoder mirrors it with transposed convolutions to a 1x1 conv."""

    def __init__(self, z_dim=32, nc=3, latent_scale=1):
        super().__init__()
        ls = int(latent_scale)
        f = 1024 * 2 * 2 * ls * ls
        enc = []
        for cin, cout in ((nc, 128), (128, 256), (256, 512), (512, 1024)):
            enc += [nn.Conv2d(cin, cout, 4, 2, 1, bias=False), nn.BatchNorm2d(cout), nn.ReLU(True)]
        self.encoder = nn.Sequential(*enc, Reshape(-1, f))
        self.fc_mu = nn.Linear(f, z_dim)
        self.fc_logvar = nn.Linear(f, z_dim)
        dec = [nn.Linear(z_dim, 1024 * 4 * 4 * ls * ls), Reshape(-1, 1024, 4 * ls, 4 * ls)]
        for cin, cout in ((1024, 512), (512, 256), (256, 128)):
            dec += [nn.ConvTranspose2d(cin, cout, 4, 2, 1, bias=False), nn.BatchNorm2d(cout), nn.ReLU(True)]
        self.decoder = nn.Sequential(*dec, nn.ConvTranspose2d(128, nc, 1))
        self.z_dim = z_dim

    def set_crop_seed(self, seed):
        self.crop_seed = seed

    def forward(self, x):
        h0, h1, w0, w1 = crop_window(self.crop_seed, x.size(2), x.size(3))
        xc = x[:, :, h0:h1, w0:w1]
        hid = self.encoder(xc)
        mu, logvar = self.fc_mu(hid), self.fc_logvar(hid)
        eps = torch.randn(*mu.size())              # the CPU generator, also when mu is on the GPU
        lat = eps.to(mu.device) * (0.5 * logvar).exp() + mu
        return xc, self.decoder(lat), lat, mu, logvar


class Discriminator(nn.Module):
    def __init__(self, z_dim=10):
        super().__init__()
        self.net = nn.Sequential(nn.Linear(z_dim, 512), nn.ReLU(True), nn.Linear(512, 512), nn.ReLU(True),
                                 nn.Linear(512, 1), nn.Sigmoid())

    def forward(self, z):
        return self.net(z)


def crop_window(seed, h, w):
    np.random.seed(seed)
    if h < CROP and w < CROP:
        return 0, CROP, 0, CROP
    if h >= CROP and w >= CROP:
        w0 = np.random.randint(w - CROP + 1)
        h0 = np.random.randint(h - CROP + 1)
        return h0, h0 + CROP, w0, w0 + CROP
    raise ValueError("Unimplemented architecture for current image size.")


def reference_query(al_set, idxs_for_query, batch_size, vae, disc, budget, device="cpu"):
    """(global indices in ascending p, query count, p in loader order) -- the loop of vaal_sampler.py:49-68."""
    loader = DataLoader(Subset(al_set, idxs_for_query), shuffle=False, batch_size=batch_size, drop_last=False)
    vae.eval()
    disc.eval()
    preds, indices = [], []
    with torch.no_grad():
        for x, _y, idxs in loader:
            _, _, _, mu, _ = vae(x.to(device))
            preds.append(disc(mu).cpu())
            indices.append(idxs.clone())
    p = torch.cat(preds).view(-1)
    count = int(min(len(idxs_for_query), budget))
    _, order = torch.topk(-p, count)
    return torch.cat(indices).numpy()[order.numpy()], count, p.numpy()


def seeded_state(module, seed):
    """Overwrite every floating-point state-dict entry of `module` (BatchNorm running statistics included) from a
    seeded recipe keyed by the entry's name and shape, so that two modules with the same layout end up identical.
    Weights are scaled by 1/sqrt(fan-in) so that activations and the discriminator's logits stay of order one."""
    sd = module.state_dict()
    for k, name in enumerate(sorted(sd)):
        t = sd[name]
        if not t.is_floating_point():
            continue
        rng = np.random.default_rng([seed, k])
        shape = tuple(t.shape)
        if name.endswith("running_var"):
            v = rng.uniform(0.5, 1.5, shape)
        elif name.endswith("running_mean") or name.endswith("bias"):
            v = rng.standard_normal(shape) * 0.1
        elif t.dim() == 1:                              # BatchNorm weight
            v = 1.0 + rng.standard_normal(shape) * 0.1
        else:
            fan_in = int(np.prod(shape[1:])) if "decoder" not in name or t.dim() == 2 else shape[0] * int(np.prod(shape[2:]))
            v = rng.standard_normal(shape) * np.sqrt(2.0 / fan_in)
        sd[name] = torch.from_numpy(v.astype(np.float32))
    module.load_state_dict(sd)
    return module


def np_rng_digest():
    st = np.random.get_state()
    return hashlib.sha256(st[1].tobytes() + repr(st[2:]).encode()).hexdigest()


def torch_rng_digest():
    return hashlib.sha256(torch.get_rng_state().numpy().tobytes()).hexdigest()


class ImagePool(torch.utils.data.Dataset):
    """al_set stand-in of seeded images: (x [3, h, w], 0, index), like custom_imagenet.py's (x, y, index)."""

    def __init__(self, n, num_classes, h, w, seed):
        self.num_classes = num_classes
        self.targets = [0] * n
        self.x = torch.from_numpy(np.random.default_rng(seed).standard_normal((n, 3, h, w)).astype(np.float32))

    def __len__(self):
        return self.x.shape[0]

    def __getitem__(self, i):
        return self.x[i], 0, i
