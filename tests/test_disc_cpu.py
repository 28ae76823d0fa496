"""PatchGAN discriminator on the CPU: the fp64 oracle (oracle/disc_oracle.py) against the golden made with the
reference's own module and autograd, the state-dict layout, argument checks, and the stride-2 dgrad's parity
decomposition."""
import json
import os

import numpy as np
import pytest
import torch

from gaussiananything_b200 import disc
from oracle import disc_oracle as do
from oracle.golden_io import load_parts

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "disc_small.npz")
KEYS = os.path.join(ROOT, "tests", "golden", "disc_keys.json")
SIZES = ("64x64", "50x70")


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


@pytest.fixture(scope="module")
def gold():
    return load_parts(GOLDEN)


@pytest.mark.parametrize("tag", SIZES)
def test_oracle_reproduces_golden(gold, tag):
    sd = disc.random_state_dict(int(gold["seed"]))
    t = tag + "/"
    r = do.d_step_grads(sd, gold[t + "real"], gold[t + "fake"])
    assert _rel(r["lr"], gold[t + "logits_real"]) < 1e-10
    assert _rel(r["lf"], gold[t + "logits_fake"]) < 1e-10
    assert abs(r["loss"] - float(gold[t + "d_loss"])) <= 1e-10 * abs(float(gold[t + "d_loss"]))
    for k, v in r["state"].items():
        if "running" in k or "num_batches" in k:
            assert _rel(v, gold[t + "state/" + k]) < 1e-10, k
    stride = int(gold["stride"])
    for k, g in r["grads"].items():
        flat = g.reshape(-1)
        assert _rel(flat[::stride], gold[t + "grad/%s/strided" % k]) < 1e-10, k
        assert abs(flat.sum() - float(gold[t + "grad/%s/sum" % k])) <= 1e-10 * np.abs(flat).sum(), k
        assert _rel(np.linalg.norm(flat), gold[t + "grad/%s/norm" % k]) < 1e-10, k
    # g-loss: -mean(fake logits) and its input gradient, on the fake call's cache
    lf = r["lf"]
    assert abs(-lf.mean() - float(gold[t + "g_loss"])) <= 1e-10
    dx, _ = do.backward(r["cache_fake"], np.full(lf.shape, -1.0 / lf.size))
    assert _rel(dx, gold[t + "grad_fake"]) < 1e-10
    # eval mode on the running statistics after both calls
    le, _, _ = do.forward(r["state"], gold[t + "real"], training=False)
    assert _rel(le, gold[t + "logits_eval"]) < 1e-10


def test_key_table_and_strict_loading():
    with open(KEYS) as f:
        keys = {k: tuple(v) for k, v in json.load(f).items()}
    m = disc.NLayerDiscriminator()
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == keys
    assert list(m.state_dict()) == list(keys)
    assert {k: tuple(v) for k, v in disc.state_dict_shapes().items()} == keys
    sd = disc.random_state_dict(1)
    m.load_state_dict(sd, strict=True)
    bad = dict(sd)
    del bad["main.3.running_var"]
    with pytest.raises(RuntimeError, match="main.3.running_var"):
        m.load_state_dict(bad, strict=True)
    bad = dict(sd, **{"main.4.weight": torch.zeros(3)})
    with pytest.raises(RuntimeError, match="main.4.weight"):
        m.load_state_dict(bad, strict=True)
    bad = dict(sd, **{"main.8.weight": torch.zeros(512, 256, 3, 3)})
    with pytest.raises(RuntimeError, match="main.8.weight"):
        m.load_state_dict(bad, strict=True)


def test_random_state_dict_draws():
    sd = disc.random_state_dict(7)
    assert torch.equal(sd["main.0.weight"], disc.random_state_dict(7)["main.0.weight"])
    assert abs(float(sd["main.8.weight"].std()) - 0.02) < 1e-3
    assert abs(float(sd["main.9.weight"].mean()) - 1.0) < 5e-3
    assert float(sd["main.9.bias"].abs().max()) == 0.0


def test_disc_flops():
    # the per-layer figures of one 512^2 image: 0.40, 4.29, 4.29, 16.65, 0.06 GFLOP
    assert disc.disc_flops(1, 512, 512) == 2 * 16 * (256 ** 2 * 3 * 64 + 128 ** 2 * 64 * 128 + 64 ** 2 * 128 * 256
                                                     + 63 ** 2 * 256 * 512 + 62 ** 2 * 512)
    assert abs(disc.disc_flops(1, 512, 512) / 1e9 - 25.7) < 0.05


@pytest.mark.parametrize("kw", [dict(input_nc=4), dict(ndf=32), dict(n_layers=4), dict(use_actnorm=True)])
def test_unsupported_arguments(kw):
    with pytest.raises(NotImplementedError):
        disc.NLayerDiscriminator(**kw)


def test_bad_inputs_raise():
    m = disc.NLayerDiscriminator()
    with pytest.raises(ValueError):
        m(torch.zeros(1, 4, 64, 64))
    with pytest.raises(ValueError):
        m(torch.zeros(2, 3, 23, 23))
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros(1, 3, 24, 24))             # the smallest input is accepted; a CPU tensor is refused


def test_sizes_follow_torch():
    for h, w in ((24, 24), (50, 70), (64, 64), (97, 33)):
        want = torch.nn.Sequential(*[torch.nn.Conv2d(1, 1, 4, s, 1) for s in disc.STRIDES])(torch.zeros(1, 1, h, w))
        assert disc.sizes(h, w)[-1] == tuple(want.shape[2:])


@pytest.mark.parametrize("H,W", [(16, 16), (17, 15), (9, 12), (2, 3)])
def test_parity_dgrad_equals_direct(H, W):
    rng = np.random.default_rng(H * 100 + W)
    Ho, Wo = do.out_size(H, 2), do.out_size(W, 2)
    g = rng.standard_normal((2, 5, Ho, Wo))
    w = rng.standard_normal((5, 3, 4, 4))
    direct = do.conv_dgrad(g, w, 2, H, W)
    assert np.allclose(do.conv_dgrad_parity(g, w, H, W), direct, rtol=0, atol=1e-12)
    # and the direct dgrad is the adjoint of the convolution
    x = rng.standard_normal((2, 3, H, W))
    assert abs((do.conv(x, w, 2) * g).sum() - (x * direct).sum()) < 1e-9


def test_dgrad_packs_match_parity_weights():
    w = torch.randn(6, 4, 4, 4)
    p1, kp1 = disc.pack_dgrad(w, 1)
    assert kp1 == 96 and p1.shape == (4, 96)
    assert torch.equal(p1.float().reshape(4, 4, 4, 6)[1, 2, 3, 5], w[5, 1, 1, 0].to(torch.bfloat16).float())
    p2, kp2 = disc.pack_dgrad(w, 2)
    assert kp2 == 24 and p2.shape == (4, 4, 24)
    for py in range(2):
        for px in range(2):
            for ty in range(2):
                for tx in range(2):
                    got = p2[2 * py + px].float().reshape(4, 2, 2, 6)[:, ty, tx, :]
                    want = w[:, :, 3 - py - 2 * ty, 3 - px - 2 * tx].t().to(torch.bfloat16).float()
                    assert torch.equal(got, want)


def test_emulation_distance_from_fp64(gold):
    """The bf16-emulating oracle's distance from fp64 on the golden inputs (the GPU tests hold the library to 1.5x
    what this measures)."""
    sd = disc.random_state_dict(int(gold["seed"]))
    for tag in SIZES:
        x = gold[tag + "/real"]
        exact, _, _ = do.forward(sd, x, True)
        emu, _, _ = do.forward(sd, x, True, emulate=True)
        assert 0 < _rel(emu, exact) < 5e-2


def test_install_shims_leaves_the_reference_discriminator():
    """The library's discriminator is slower than bf16 cuDNN, so install_shims() does not replace the reference's."""
    import sys
    import types

    import gaussiananything_b200 as ga
    name = "nsr.losses.disc"
    old = sys.modules.get(name)
    stand_in = types.ModuleType(name)
    stand_in.NLayerDiscriminator = object
    sys.modules[name] = stand_in
    try:
        ga.install_shims()
        assert getattr(sys.modules[name], "NLayerDiscriminator") is object
    finally:
        if old is None:
            del sys.modules[name]
        else:
            sys.modules[name] = old


def test_cumulative_momentum_is_refused():
    m = disc.NLayerDiscriminator()
    m.main[6].momentum = None
    with pytest.raises(NotImplementedError, match="momentum"):
        m(torch.zeros(1, 3, 32, 32))
