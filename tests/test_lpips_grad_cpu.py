"""LPIPS backward references on the CPU: the fp64 oracle against the reference's own autograd (golden), the
bf16-emulating backward against autograd through the emulating forward, the zero-vector rule, and the install_shims
hook for nsr.losses.builder.LPIPSLoss."""
import os
import sys
import types

import pytest
import torch
import torch.nn.functional as F

from oracle import lpips_oracle as lo
from oracle.golden_io import load_parts
from tests import lpips_grad_ref as lg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "lpips_grad_small.npz")
INPUTS = os.path.join(ROOT, "tests", "golden", "lpips_small.npz")
SIZES = ("64x64", "50x70")
# The hand-written emulated backward against autograd through the emulating forward.  The two round at the same
# points except that autograd also rounds the packed input's gradient to bf16 (its cast) and runs the head in fp64;
# the last-bit differences that follows flip some bf16 roundings further down.  Measured up to 5.5e-3 per image.
TOL_EMU_AUTOGRAD = 6e-3


@pytest.fixture(scope="module")
def golden():
    g = load_parts(GOLDEN)
    z = load_parts(INPUTS)
    for s in SIZES:
        g[s + "/in0"], g[s + "/in1"] = z[s + "/in0"], z[s + "/in1"]
    return g


@pytest.mark.parametrize("size", SIZES)
def test_fp64_oracle_reproduces_the_reference_autograd(golden, size):
    sd = lo.random_state_dict(int(golden["seed"]))
    a, b = torch.from_numpy(golden[size + "/in0"]), torch.from_numpy(golden[size + "/in1"])
    g = torch.from_numpy(golden[size + "/g"])
    assert float(g.abs().min()) == 0.0
    d0, d1 = lg.lpips_grad(sd, a, b, g)
    for d, key in ((d0, "/grad0"), (d1, "/grad1")):
        want = torch.from_numpy(golden[size + key])
        e = lg.rel_l2(d, want)
        print(size, key, "rel-L2 per image", e.tolist())
        nz = g != 0
        assert float(e[nz].max()) <= 1e-10
        assert torch.all(d[~nz] == 0) and torch.all(want[~nz] == 0)
    only1 = lg.lpips_grad(sd, a, b, g, sides=(1,))
    assert only1[0] is None and torch.equal(only1[1], d1)


@pytest.mark.parametrize("size", SIZES)
def test_emulated_backward_against_autograd_through_the_emulated_forward(golden, size):
    sd = lo.random_state_dict(0)
    a, b = torch.from_numpy(golden[size + "/in0"]), torch.from_numpy(golden[size + "/in1"])
    g = torch.tensor([0.75, -1.25, 0.5, 2.0])
    emu = lg.lpips_grad(sd, a, b, g, emulate_bf16=True)
    ag = lg.emulated_autograd(sd, a, b, g)
    f64 = lg.lpips_grad(sd, a, b, g)
    for s in range(2):
        e = lg.rel_l2(emu[s], ag[s])
        e64 = lg.rel_l2(emu[s], f64[s])
        print(size, "side", s, "emulated vs autograd", e.tolist(), "vs fp64", e64.tolist())
        assert float(e.max()) <= TOL_EMU_AUTOGRAD
        assert torch.all(torch.isfinite(emu[s]))


def test_emulated_backward_swaps_with_the_images(golden):
    sd = lo.random_state_dict(0)
    a, b = torch.from_numpy(golden["64x64/in0"]), torch.from_numpy(golden["64x64/in1"])
    g = torch.tensor([0.75, -1.25, 0.5, 2.0])
    ab, ba = lg.lpips_grad(sd, a, b, g, emulate_bf16=True), lg.lpips_grad(sd, b, a, g, emulate_bf16=True)
    assert torch.equal(ab[0], ba[1]) and torch.equal(ab[1], ba[0])
    same = lg.lpips_grad(sd, a, a, g, emulate_bf16=True)
    assert torch.all(same[0] == 0) and torch.all(same[1] == 0)


def test_zero_vector_rule():
    """Where a tap's feature vector is all zero the head gradient is 0, never NaN.  The reference's normalize_tensor
    gives NaN there; its ReLU backward (a select) turns that into 0, so through the ReLU both agree."""
    g = torch.Generator().manual_seed(5)
    z = torch.randn(2, 16, 5, 6, generator=g, dtype=torch.float64)
    z[0, :, 2, 3] = -torch.rand(16, generator=g, dtype=torch.float64) - 0.1     # this pixel's ReLU output is all 0
    z[1, :, 0, 0] = -1.0
    zo = torch.randn(2, 16, 5, 6, generator=g, dtype=torch.float64)
    lin = torch.rand(16, generator=g, dtype=torch.float64)
    gp = torch.tensor([0.7, -1.1], dtype=torch.float64)
    # the reference's head on relu(z), autograd to z
    zr = z.clone().requires_grad_(True)
    f, fo = F.relu(zr), F.relu(zo)
    norm = lambda t: t / (t.pow(2).sum(1, keepdim=True).sqrt() + 1e-10)
    val = ((norm(f) - norm(fo)) ** 2 * lin.reshape(1, -1, 1, 1)).sum(1).mean((1, 2))
    want = torch.autograd.grad((val * gp).sum(), zr)[0]
    assert torch.all(torch.isfinite(want))
    head = lg.head_grad(f.detach().float(), fo.float(), lin.float(), gp.float())
    assert torch.all(torch.isfinite(head))
    assert torch.all(head[0, :, 2, 3] == 0) and torch.all(head[1, :, 0, 0] == 0)
    got = torch.where(f.detach() > 0, head.double(), torch.zeros((), dtype=torch.float64))
    assert float((got - want).abs().max()) <= 1e-6 * float(want.abs().max())


def _with_modules(names, fn):
    keep = ("diff_surfel_rasterization", "transport", "transport.transport", "transport.path", "transport.integrators")
    saved = {k: sys.modules.get(k) for k in names + keep}
    try:
        fn()
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def test_install_shims_sets_lpips_loss():
    import gaussiananything_b200 as ga
    from gaussiananything_b200 import lpips
    names = ("nsr", "nsr.losses", "nsr.losses.builder")

    def run():
        for n in names:
            sys.modules[n] = types.ModuleType(n)
        sentinel = object()
        sys.modules["nsr.losses.builder"].LPIPSLoss = sentinel
        ga.install_shims()
        assert sys.modules["nsr.losses.builder"].LPIPSLoss is lpips.LPIPSLoss
    _with_modules(names, run)


def test_install_shims_without_the_loss_module():
    import gaussiananything_b200 as ga
    names = ("nsr.losses.builder",)

    def run():
        sys.modules.pop("nsr.losses.builder", None)
        ga.install_shims()
        assert "nsr.losses.builder" not in sys.modules
    _with_modules(names, run)


def test_loss_module_interface():
    """LPIPSLoss keeps the reference's constructor arguments and takes an existing LPIPS without building one."""
    from gaussiananything_b200 import lpips

    class Stub:
        def values(self, in0, in1, normalize=False):
            return (in0 - in1).abs().mean((1, 2, 3)).reshape(-1, 1, 1, 1)
    loss = lpips.LPIPSLoss(loss_weight=0.8, use_input_norm=True, range_norm=True, lpips=Stub())
    p, t = torch.zeros(2, 3, 4, 4), torch.ones(2, 3, 4, 4)
    out = loss(p, t, conf_sigma_percl=None)
    assert out.dim() == 0 and float(out) == pytest.approx(0.8)
