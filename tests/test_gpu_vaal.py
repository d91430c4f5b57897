"""K9 / VAALSampler on the H100: logits against an fp64 evaluation of the discriminator under the K3 bar (1e-5 of the
magnitude chain), bit-equal p for equal rows with ties resolved by pool position, argument checks, and the whole query
on the reference's goldens (picks and RNG states)."""
import ctypes
import os
import re
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

import vaal_oracle as V

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def eng():
    from active_learning_b200.engine import Engine
    return Engine()


@pytest.fixture
def no_tf32():
    """cuDNN and cuBLAS in full fp32 for the golden query: the goldens were taken in fp32 on the CPU."""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _disc(z, seed):
    return V.seeded_state(V.Discriminator(z_dim=z), seed)


def _fp64(mu, disc):
    """(logits, magnitude chain) in fp64: |b3| + |w3|.(|b2| + |W2|.(|b1| + |W1|.|mu|))."""
    l1, l2, l3 = disc.net[0], disc.net[2], disc.net[4]
    W = [t.detach().double().cuda() for t in (l1.weight, l1.bias, l2.weight, l2.bias, l3.weight, l3.bias)]
    x = mu.double()
    h1 = torch.relu(x @ W[0].T + W[1])
    h2 = torch.relu(h1 @ W[2].T + W[3])
    lg = (h2 @ W[4].T + W[5]).view(-1)
    c1 = x.abs() @ W[0].abs().T + W[1].abs()
    c2 = c1 @ W[2].abs().T + W[3].abs()
    chain = (c2 @ W[4].abs().T + W[5].abs()).view(-1)
    return lg, chain


@pytest.mark.parametrize("z", [32, 64, 100])
@pytest.mark.parametrize("n", [1, 127, 128, 129, 131073])
def test_k9_logits_within_the_k3_bar(eng, n, z):
    disc = _disc(z, 10 * z + 1)
    g = torch.Generator(device="cuda").manual_seed(n + z)
    ld = ((z + 3) & ~3) + 4                                 # a padded leading dimension
    slab = torch.randn(n, ld, device="cuda", generator=g)
    mu = slab[:, :z]
    p, lg = eng.vaal_scores(slab, disc, return_logits=True)
    ref, chain = _fp64(mu, disc)
    err = (lg.double() - ref).abs()
    assert bool((err <= 1e-5 * chain).all()), float((err / chain).max())
    # the sigmoid on top: fp32 rounding of a value in (0, 1) plus the logit error through sigmoid' <= 1/4
    pref = torch.sigmoid(ref)
    assert bool(((p.double() - pref).abs() <= 0.25 * 1e-5 * chain + 2e-7).all())
    # the same rows at ld = z (a copy into a padded slab inside the engine when z % 4 != 0)
    p2 = eng.vaal_scores(mu.contiguous(), disc)
    assert torch.equal(p2, p)


def test_equal_rows_give_equal_p_and_ties_go_by_pool_position(eng):
    disc = _disc(64, 5)
    rng = np.random.default_rng(0)
    base = torch.randn(300, 64, device="cuda")
    which = torch.from_numpy(rng.integers(0, 300, 20000)).cuda()
    mu = base[which].contiguous()
    p = eng.vaal_scores(mu, disc)
    first = eng.vaal_scores(base, disc)
    assert torch.equal(p, first[which])                       # bit-equal whatever the row's tile, CTA or slice
    b = 4000
    pos = eng.select_smallest(p, b).cpu().numpy()
    ph = p.cpu().numpy()
    assert pos.tolist() == np.argsort(ph, kind="stable")[:b].tolist()


def test_invalid_arguments_are_rejected(eng):
    from active_learning_b200 import _lib
    from active_learning_b200._lib import AlqError
    lib = eng.lib
    z = 64
    mu = torch.randn(256, z, device="cuda")
    w1, b1 = torch.randn(512, z, device="cuda"), torch.randn(512, device="cuda")
    w2, b2 = torch.randn(512, 512, device="cuda"), torch.randn(512, device="cuda")
    w3, b3 = torch.randn(512, device="cuda"), torch.randn(1, device="cuda")
    p = torch.empty(256, device="cuda")
    P = lambda t, off=0: ctypes.c_void_p(t.data_ptr() + off)  # noqa: E731
    st = eng._stream()

    def call(n=256, zz=z, ldmu=z, ldw1=z, ldw2=512, hidden=512, mu_off=0, w1p=None):
        return lib.alq_vaal_scores(eng._h, P(mu, mu_off), n, zz, ldmu, w1p if w1p is not None else P(w1), ldw1, P(b1),
                                   P(w2), ldw2, P(b2), P(w3), P(b3), hidden, P(p), None, st)

    assert call() == 0
    torch.cuda.synchronize()
    for kw in (dict(hidden=256), dict(hidden=1024), dict(ldmu=z - 4), dict(ldmu=66), dict(ldw1=62), dict(ldw2=510),
               dict(ldw2=511), dict(mu_off=4), dict(zz=0), dict(n=-1), dict(w1p=ctypes.c_void_p(0))):
        assert call(**kw) == 1, kw                              # ALQ_ERR_INVALID
    assert _lib.ERR_NAMES[1] == "ALQ_ERR_INVALID"
    with pytest.raises(AlqError):
        eng.vaal_scores(mu[:, :10], _disc(z, 1))                 # fewer columns than the discriminator's z
    with pytest.raises(AlqError):
        eng.vaal_scores(mu.cpu(), _disc(z, 1))
    with pytest.raises(AlqError):
        eng.vaal_scores(mu, torch.nn.Sequential(torch.nn.Linear(z, 512), torch.nn.ReLU()))
    assert eng.vaal_scores(mu[:0], _disc(z, 1)).numel() == 0


@pytest.mark.parametrize("tag", ["a", "b", "c"])
def test_query_replays_the_reference_goldens(eng, no_tf32, tag):
    from test_vaal import fixture_sampler, golden_query, load_gold
    gold = load_gold()
    s, budget = fixture_sampler(gold, tag, eng)
    idx, cost, np_d, torch_d = golden_query(gold, s, budget)
    assert isinstance(idx, np.ndarray) and idx.dtype == np.int64
    assert idx.tolist() == gold[f"{tag}_picks"].tolist() and cost == int(gold[f"{tag}_cost"])
    assert np_d == str(gold[f"{tag}_np_digest"]) and torch_d == str(gold[f"{tag}_torch_digest"])
    assert not (s.net.training or s.vae.training or s.discriminator.training)


def test_k9_compiles_without_spills():
    """ptxas's register and spill report of K9 for sm_90a (printed with -s)."""
    import shutil
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    src = os.path.join(os.path.dirname(HERE), "active_learning_b200", "csrc", "alq_vaal.cu")
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                            "-c", src, "-o", os.path.join(tmp, "k9.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    report = re.findall(r"Compiling entry function '(\w*vaal_layer_kernel\w*)'.*?(\d+) bytes spill stores, (\d+) bytes spill "
                        r"loads.*?Used (\d+) registers", r.stderr, flags=re.S)
    assert len(report) == 2
    for name, stores, loads, regs in report:
        print(f"{name}: {regs} registers, spills {stores} B stored / {loads} B loaded", file=sys.stderr)
        assert stores == loads == "0"
