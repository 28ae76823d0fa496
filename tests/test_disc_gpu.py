"""PatchGAN discriminator on the GPU (include/ga_b200.h Part 11, gaussiananything_b200.disc): forward in training and
eval mode, running statistics, input and parameter gradients against the bf16-emulating oracle and the fp64 golden,
frozen parameters and detached inputs, accumulation, the reference's d-step, AdamW steps against a torch PatchGAN,
and determinism.

Bounds: the bf16-emulating oracle's own distance from fp64 is measured on the CPU for the same case, and the GPU is
held to 1.5 times it (as LPIPS's are); the emulation rounds where the kernels round, with every sum in fp64."""
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

from gaussiananything_b200 import disc
from oracle import disc_oracle as do
from oracle.golden_io import load_parts

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "disc_small.npz")
SIZES = ("64x64", "50x70")
RATIO = 1.5
# fp32 rounding of sums the emulation forms exactly (the bias gradients, .grad accumulation over two calls)
FLOOR = 1e-5


def _rel(a, b):
    a = a.detach().double().cpu().numpy() if torch.is_tensor(a) else np.asarray(a, np.float64)
    b = b.detach().double().cpu().numpy() if torch.is_tensor(b) else np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


@pytest.fixture(scope="module")
def gold():
    return load_parts(GOLDEN)


def _model(seed, train=True):
    m = disc.NLayerDiscriminator()
    m.load_state_dict(disc.random_state_dict(seed), strict=True)
    return m.to(DEV).train(train)


def _bound(emu, exact):
    return RATIO * _rel(emu, exact) + FLOOR


@pytest.mark.parametrize("tag", SIZES)
def test_forward_train_eval_and_running_stats(gold, tag):
    t = tag + "/"
    seed = int(gold["seed"])
    sd = disc.random_state_dict(seed)
    emu = do.d_step_grads(sd, gold[t + "real"], gold[t + "fake"], emulate=True)
    m = _model(seed)
    real, fake = torch.tensor(gold[t + "real"], device=DEV), torch.tensor(gold[t + "fake"], device=DEV)
    with torch.no_grad():
        lr, lf = m(real), m(fake)
    for got, e, g64 in ((lr, emu["lr"], gold[t + "logits_real"]), (lf, emu["lf"], gold[t + "logits_fake"])):
        assert got.dtype == torch.float32 and tuple(got.shape) == g64.shape
        b = _bound(e, g64)
        assert _rel(got, g64) <= b, (_rel(got, g64), b)
        assert _rel(got, e) <= b, (_rel(got, e), b)
    sdm = m.state_dict()
    for k, v in emu["state"].items():
        if "num_batches" in k:
            assert int(sdm[k]) == 2
        elif "running" in k:
            b = _bound(v, gold[t + "state/" + k])
            assert _rel(sdm[k], gold[t + "state/" + k]) <= b, k
    m.eval()
    with torch.no_grad():
        le = m(real)
    le_emu, _, _ = do.forward(emu["state"], gold[t + "real"], training=False, emulate=True)
    b = _bound(le_emu, gold[t + "logits_eval"])
    assert _rel(le, gold[t + "logits_eval"]) <= b, (_rel(le, gold[t + "logits_eval"]), b)


@pytest.mark.parametrize("tag", SIZES)
def test_gradients_match_oracle(gold, tag):
    t = tag + "/"
    seed = int(gold["seed"])
    sd = disc.random_state_dict(seed)
    exact = do.d_step_grads(sd, gold[t + "real"], gold[t + "fake"])
    emu = do.d_step_grads(sd, gold[t + "real"], gold[t + "fake"], emulate=True)
    m = _model(seed)
    real = torch.tensor(gold[t + "real"], device=DEV)
    fake = torch.tensor(gold[t + "fake"], device=DEV).requires_grad_(True)
    lr = m(real)
    lf = m(fake)
    d_loss = 0.5 * (torch.relu(1.0 - lr).mean() + torch.relu(1.0 + lf).mean())
    d_loss.backward(retain_graph=False)
    for k, p in m.named_parameters():
        b = _bound(emu["grads"][k], exact["grads"][k])
        assert p.grad is not None and p.grad.shape == p.shape
        assert _rel(p.grad, exact["grads"][k]) <= b, (k, _rel(p.grad, exact["grads"][k]), b)
    # the input gradient of the g-loss -mean(D(fake)) (a fresh train-mode call on the same weights)
    m2 = _model(seed)
    fake2 = torch.tensor(gold[t + "fake"], device=DEV).requires_grad_(True)
    (-m2(fake2).mean()).backward()
    lf_e = emu["lf"]
    dx_emu, _ = do.backward(emu["cache_fake"], np.full(lf_e.shape, -1.0 / lf_e.size))
    b = _bound(dx_emu, gold[t + "grad_fake"])
    assert _rel(fake2.grad, gold[t + "grad_fake"]) <= b, (_rel(fake2.grad, gold[t + "grad_fake"]), b)


def test_large_batch_512(gold):
    """4 x 512^2 in training mode: logits and the parameter gradients of sum(logits * g) against the emulation."""
    torch.manual_seed(0)
    x = (torch.rand(4, 3, 512, 512) * 2 - 1)
    seed = 5
    sd = disc.random_state_dict(seed)
    lo, cache, new = do.forward(sd, x.numpy(), True, emulate=True)
    lo64, cache64, _ = do.forward(sd, x.numpy(), True)
    g = np.random.default_rng(1).standard_normal(lo.shape) / lo.size
    _, ge = do.backward(cache, g)
    _, g64 = do.backward(cache64, g)
    m = _model(seed)
    out = m(x.to(DEV))
    assert _rel(out, lo64) <= _bound(lo, lo64)
    (out * torch.tensor(g, device=DEV, dtype=torch.float32)).sum().backward()
    for k, p in m.named_parameters():
        assert _rel(p.grad, g64[k]) <= _bound(ge[k], g64[k]), (k, _rel(p.grad, g64[k]), _bound(ge[k], g64[k]))
    sdm = m.state_dict()
    for k, v in new.items():
        if "running" in k:
            assert _rel(sdm[k], v) < 1e-3, k


def test_frozen_parameters_and_detached_input(gold):
    m = _model(3)
    for p in m.parameters():
        p.requires_grad_(False)
    x = torch.tensor(gold["64x64/fake"], device=DEV).requires_grad_(True)
    (-m(x).mean()).backward()
    assert x.grad is not None and torch.isfinite(x.grad).all()
    assert all(p.grad is None for p in m.parameters())
    # only conv 3 trainable, input detached: only conv 3 gets a gradient
    m.main[5].weight.requires_grad_(True)
    y = torch.tensor(gold["64x64/real"], device=DEV)
    m(y).mean().backward()
    assert m.main[5].weight.grad is not None
    assert all(p.grad is None for n, p in m.named_parameters() if n != "main.5.weight")
    assert not y.requires_grad and y.grad is None


def test_gradients_accumulate_and_are_deterministic(gold):
    x = torch.tensor(gold["50x70/real"], device=DEV)

    def run():
        m = _model(9)
        xi = x.clone().requires_grad_(True)
        out = m(xi)
        out.square().mean().backward()
        return m, out.detach().clone(), xi.grad.clone()

    m1, o1, gx1 = run()
    m2, o2, gx2 = run()
    assert torch.equal(o1, o2) and torch.equal(gx1, gx2)
    for (k, p1), p2 in zip(m1.named_parameters(), m2.parameters()):
        assert torch.equal(p1.grad, p2.grad), k
    for (k, b1), b2 in zip(m1.named_buffers(), m2.buffers()):
        assert torch.equal(b1, b2), k
    first = {k: p.grad.clone() for k, p in m1.named_parameters()}
    m1(x).square().mean().backward()
    for k, p in m1.named_parameters():
        # the second call normalises with the same batch statistics, so it adds the same gradient
        assert torch.allclose(p.grad, 2 * first[k], rtol=1e-5, atol=1e-12), k


def test_d_step_fills_only_parameter_gradients(gold):
    m = _model(11)
    real = torch.tensor(gold["64x64/real"], device=DEV)
    fake = torch.tensor(gold["64x64/fake"], device=DEV, requires_grad=True).detach()
    lr = m(real)
    lf = m(fake)
    (0.5 * (torch.relu(1.0 - lr).mean() + torch.relu(1.0 + lf).mean())).backward()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in m.parameters())
    assert real.grad is None and fake.grad is None
    assert int(m.main[3].num_batches_tracked) == 2


def _torch_patchgan():
    c = disc.CHANNELS
    return nn.Sequential(
        nn.Conv2d(c[0], c[1], 4, 2, 1), nn.LeakyReLU(0.2, True),
        nn.Conv2d(c[1], c[2], 4, 2, 1, bias=False), nn.BatchNorm2d(c[2]), nn.LeakyReLU(0.2, True),
        nn.Conv2d(c[2], c[3], 4, 2, 1, bias=False), nn.BatchNorm2d(c[3]), nn.LeakyReLU(0.2, True),
        nn.Conv2d(c[3], c[4], 4, 1, 1, bias=False), nn.BatchNorm2d(c[4]), nn.LeakyReLU(0.2, True),
        nn.Conv2d(c[4], c[5], 4, 1, 1))


def test_adamw_d_steps_track_torch(gold):
    """Five AdamW d-steps (betas (0, 0.999), as the reference's trainer) from one state on the library, on an fp32
    torch PatchGAN and on the same PatchGAN under bf16 autocast.  Adam's normalised steps turn gradient noise into
    full-size steps, so the yardstick is measured in the same run: the library stays within 1.5 times the bf16
    autocast run's distance from fp32, in the weights and in the logits afterwards."""
    sd = disc.random_state_dict(13)
    lib = _model(13)
    nets = [lib]
    for _ in range(2):
        ref = _torch_patchgan()
        ref.load_state_dict({k[len("main."):]: v for k, v in sd.items()}, strict=True)
        nets.append(ref.to(DEV).train())
    amps = (False, False, True)
    opts = [torch.optim.AdamW(m.parameters(), lr=2e-4, betas=(0.0, 0.999)) for m in nets]
    real = torch.tensor(gold["64x64/real"], device=DEV)
    fake = torch.tensor(gold["64x64/fake"], device=DEV)
    with torch.backends.cudnn.flags(enabled=True, deterministic=True, allow_tf32=False):
        for step in range(5):
            for m, opt, amp in zip(nets, opts, amps):
                opt.zero_grad(set_to_none=True)
                with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
                    lr, lf = m(real).float(), m(fake).float()
                (0.5 * (torch.relu(1.0 - lr).mean() + torch.relu(1.0 + lf).mean())).backward()
                opt.step()
        vec = lambda m: torch.cat([p.detach().reshape(-1) for p in m.parameters()])
        p0 = torch.cat([sd[k].reshape(-1) for k, _ in lib.named_parameters()]).to(DEV)
        moved = float((vec(nets[1]) - p0).norm())
        d_lib = float((vec(lib) - vec(nets[1])).norm()) / moved
        d_b16 = float((vec(nets[2]) - vec(nets[1])).norm()) / moved
        for m in nets:
            m.eval()
        with torch.no_grad():
            lo = [m(real).float() for m in nets[:2]]
            with torch.autocast("cuda", dtype=torch.bfloat16):
                lo.append(nets[2](real).float())
    e_lib, e_b16 = _rel(lo[0], lo[1]), _rel(lo[2], lo[1])
    print("AdamW 5 steps: weights %.3g (bf16 autocast %.3g) of the fp32 run's movement; logits %.3g (bf16 %.3g)"
          % (d_lib, d_b16, e_lib, e_b16))
    assert d_lib <= RATIO * d_b16 + FLOOR
    assert e_lib <= RATIO * e_b16 + FLOOR


def test_bf16_input_and_gradient_dtype(gold):
    """The input is rounded to bf16 by the pack either way, so a bf16 input gives the fp32 path's bits, and its
    gradient comes back in bf16."""
    x32 = torch.tensor(gold["64x64/fake"], device=DEV).to(torch.bfloat16).float().requires_grad_(True)
    x16 = x32.detach().to(torch.bfloat16).requires_grad_(True)
    m1, m2 = _model(21), _model(21)
    o32, o16 = m1(x32), m2(x16)
    assert o16.dtype == torch.float32 and torch.equal(o32, o16)
    (-o32.mean()).backward()
    (-o16.mean()).backward()
    assert x16.grad.dtype == torch.bfloat16 and torch.equal(x16.grad, x32.grad.to(torch.bfloat16))
    with torch.autocast("cuda", dtype=torch.bfloat16):
        assert torch.equal(m1.eval()(x16), m2.eval()(x16))


def test_non_fp32_parameters_and_buffers_raise(gold):
    x = torch.tensor(gold["64x64/real"], device=DEV)
    m = _model(22)
    m.main[5].weight.data = m.main[5].weight.data.half()
    with pytest.raises(RuntimeError, match="fp32"):
        m(x)
    m = _model(22)
    m.main[9].running_var = m.main[9].running_var.double()
    with pytest.raises(RuntimeError, match="fp32"):
        m(x)
    m = _model(22).cpu()
    with pytest.raises(RuntimeError):
        m(x)


def test_parameter_changed_before_backward_raises(gold):
    m = _model(23)
    out = m(torch.tensor(gold["64x64/real"], device=DEV))
    with torch.no_grad():
        m.main[8].weight.add_(1e-3)              # an optimiser step between forward and backward
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        out.mean().backward()


def test_second_backward_through_one_call_raises(gold):
    m = _model(24)
    out = m(torch.tensor(gold["64x64/real"], device=DEV))
    out.mean().backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="second backward"):
        out.mean().backward()


def test_g_step_through_the_rasteriser_to_gauss13():
    """The reference's g-step: surfels rendered by GaussianRenderer2DGS at 64^2, the image (its layout and dtype as the
    renderer gives them) through the discriminator in training mode, -mean(logits) back to a finite gauss13.grad.
    The image gradient the discriminator returns is the one the rasteriser's backward consumes."""
    from gaussiananything_b200.gs_surfel import GaussianRenderer2DGS
    from tests.helpers import cameras, scene
    H, V = 64, 4
    vs, ps, cs, tf = cameras(V)
    g13 = torch.tensor(scene(2000, 5, 3.0), device=DEV)[None].contiguous().requires_grad_(True)
    view, proj = torch.tensor(vs, device=DEV)[None], torch.tensor(ps, device=DEV)[None]
    pos = torch.tensor(cs, device=DEV)[None]
    r = GaussianRenderer2DGS(H, 3, {})
    out = r.render(g13, view, proj, pos, tf)
    image = out["image"][0]                                   # [V, 3, H, W]
    m = _model(25)
    for p in m.parameters():
        p.requires_grad_(False)                               # the g-step does not train the discriminator
    loss = -m(image * 2 - 1).mean()
    seen = []
    image.register_hook(lambda g: seen.append(g.detach().clone()))
    loss.backward(retain_graph=True)                          # keeps the renderer's graph for the check below
    g_img = seen[0]
    assert torch.isfinite(g_img).all() and torch.any(g_img != 0)
    want = torch.autograd.grad([image], g13, [g_img])[0]
    assert torch.isfinite(g13.grad).all() and torch.any(g13.grad != 0)
    assert float((g13.grad - want).abs().max()) <= 1e-5 * float(want.abs().max())
    assert all(p.grad is None for p in m.parameters())
