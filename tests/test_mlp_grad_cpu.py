"""CPU checks of the differentiable FusedMLP (include/ga_b200.h Part 13): the fp64 reference against torch autograd,
where the bf16 emulation rounds, every refusal, the host-only argument check of the C library, the state-dict layout
of xformers' FusedMLP and the opt-in shim."""
import ctypes as C
import json
import os
import sys
import types

import pytest
import torch

from tests import mlp_grad_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _case(M, D, Hd, seed, bf16_values=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, D, generator=g, dtype=torch.float64)
    w1 = (torch.rand(Hd, D, generator=g, dtype=torch.float64) * 2 - 1) / D ** 0.5
    b1 = 0.1 * torch.randn(Hd, generator=g, dtype=torch.float64)
    w2 = (torch.rand(D, Hd, generator=g, dtype=torch.float64) * 2 - 1) / Hd ** 0.5
    b2 = 0.1 * torch.randn(D, generator=g, dtype=torch.float64)
    dy = torch.randn(M, D, generator=g, dtype=torch.float64)
    if bf16_values:
        x, w1, w2, dy = (R.bf16(t) for t in (x, w1, w2, dy))
    return x, w1, b1, w2, b2, dy


@pytest.mark.parametrize("M,D,Hd", [(5, 8, 32), (37, 24, 96), (64, 64, 256)])
def test_fp64_reference_matches_autograd(M, D, Hd):
    args = _case(M, D, Hd, seed=M)
    ref, auto = R.mlp(*args), R.mlp_autograd(*args)
    for k in ("y", "dx", "dW1", "db1", "dW2", "db2"):
        assert R.rel_l2(ref[k], auto[k]) < 1e-13, k


def test_emulation_rounds_where_the_header_says():
    x, w1, b1, w2, b2, dy = _case(50, 32, 128, seed=3, bf16_values=True)
    ref, emu = R.mlp(x, w1, b1, w2, b2, dy), R.mlp(x, w1, b1, w2, b2, dy, emulate=True)
    # bf16-valued operands: the emulation's products are the fp64 ones
    assert torch.equal(emu["v"], ref["v"]) and torch.equal(emu["dW2"][:, :0], ref["dW2"][:, :0])
    assert torch.equal(emu["Z"], R.bf16(ref["v"]))                       # Z = bf16(v)
    assert torch.equal(emu["H"], R.bf16(R.gelu(ref["v"])))               # H = bf16(gelu(v)), from the unrounded v
    assert torch.equal(emu["dZ"], R.bf16(emu["dH"] * R.gelu_grad(emu["Z"])))   # gelu' at the bf16 Z
    assert torch.equal(emu["db1"], emu["dZ"].sum(0))                     # db1 sums the bf16 dZ
    assert torch.equal(emu["dW2"], dy.T @ emu["H"]) and torch.equal(emu["dx"], emu["dZ"] @ w1)
    for k in ("Z", "H", "dZ"):
        assert torch.equal(emu[k], R.bf16(emu[k])), k
    # and it is not the fp64 result
    for k in ("Z", "H", "dZ", "dx", "dW1"):
        assert R.rel_l2(emu[k], ref[k]) > 1e-4, k


def test_emulation_distance_is_the_documented_size():
    x, w1, b1, w2, b2, dy = _case(300, 64, 256, seed=0)
    ref, emu = R.mlp(x, w1, b1, w2, b2, dy), R.mlp(x, w1, b1, w2, b2, dy, emulate=True)
    for k in ("H", "Z", "y", "dZ", "dx", "dW1", "dW2", "db1"):
        assert 1e-4 < R.rel_l2(emu[k], ref[k]) < 1e-2, k


# ---- refusals -------------------------------------------------------------------------------------------------------

def _mlp():
    from gaussiananything_b200 import mlp
    return mlp


@pytest.mark.parametrize("kw,exc", [
    (dict(dropout=0.1), NotImplementedError),
    (dict(activation="relu"), NotImplementedError),
    (dict(activation="squared_relu"), NotImplementedError),
    (dict(bias=False), NotImplementedError),
    (dict(dim_model=100), NotImplementedError),                  # D % 8
    (dict(dim_model=4, hidden_layer_multiplier=4), NotImplementedError),   # D < 8
    (dict(dim_model=24, hidden_layer_multiplier=1.5), NotImplementedError),   # hidden 36
])
def test_fused_mlp_refusals(kw, exc):
    args = dict(dim_model=64, dropout=0.0, activation="gelu", hidden_layer_multiplier=4)
    args.update(kw)
    with pytest.raises(exc):
        _mlp().FusedMLP(**args)


def test_fused_mlp_accepts_gelu_spellings():
    M = _mlp()

    class Activation(str):          # xformers' Activation is a str Enum with value "gelu"
        value = "gelu"
    for act in ("gelu", "GeLU", Activation("GeLU")):
        assert isinstance(M.FusedMLP(64, 0.0, act, 4), torch.nn.Module)
    assert M.FusedMLP(64, 0, "gelu", 4, True, "extra", foo=1).mlp[0].weight.shape == (256, 64)


def test_cpu_tensors_raise():
    M = _mlp()
    m = M.FusedMLP(64, 0.0, "gelu", 4)
    x = torch.randn(3, 64)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m(x)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        M.linear(x, torch.randn(16, 64), torch.randn(16))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        M.fused_mlp(x, *[p.detach() for p in m.parameters()])


def test_function_shape_and_width_refusals():
    M = _mlp()
    x = torch.randn(3, 64)
    with pytest.raises(ValueError):
        M.linear(x, torch.randn(16, 32))
    with pytest.raises(ValueError):
        M.linear(x, torch.randn(16, 64), torch.randn(8))
    with pytest.raises(TypeError):
        M.linear(x.double(), torch.randn(16, 64))


def test_parameters_follow_nn_linear_init_and_zero_biases():
    torch.manual_seed(0)
    m = _mlp().FusedMLP(256, 0.0, "gelu", 4)
    w1, b1, w2, b2 = m.mlp[0].weight, m.mlp[1].bias, m.mlp[2].weight, m.mlp[3].bias
    assert all(p.dtype == torch.float32 for p in (w1, b1, w2, b2))
    assert not b1.detach().any() and not b2.detach().any()
    # kaiming_uniform(a = sqrt(5)): U(-1/sqrt(fan_in), 1/sqrt(fan_in))
    w1m, w2m = float(w1.detach().abs().max()), float(w2.detach().abs().max())
    assert 0.9 / 16 < w1m <= 1 / 16 and 0.9 / 32 < w2m <= 1 / 32


@pytest.mark.parametrize("model,D", [("DiT-PixArt-PCD-CLAY-B", 768), ("DiT-PixArt-PCD-CLAY-L", 1024)])
def test_state_dict_is_xformers_fused_mlp(model, D):
    keys = json.load(open(os.path.join(ROOT, "tests", "golden", "dit_state_dict_keys.json")))[model]
    pre = "blocks.0.mlp."
    want = {k[len(pre):]: tuple(v) for k, v in keys.items() if k.startswith(pre)}
    m = _mlp().FusedMLP(dim_model=D, dropout=0, activation="gelu", hidden_layer_multiplier=4)
    got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert got == want
    sd = {k: torch.randn(v) for k, v in want.items()}
    m.load_state_dict(sd, strict=True)
    assert torch.equal(m.mlp[2].weight, sd["mlp.2.weight"])


# ---- shim -----------------------------------------------------------------------------------------------------------

_XF = ("xformers", "xformers.components", "xformers.components.feedforward", "xformers.components.feedforward.fused_mlp")


@pytest.fixture
def saved_xformers():
    saved = {k: sys.modules.get(k) for k in _XF}
    yield
    for k, v in saved.items():
        if v is None:
            sys.modules.pop(k, None)
        else:
            sys.modules[k] = v


def test_install_shims_sets_fused_mlp_on_a_stub(saved_xformers):
    M = _mlp()
    mods = {}
    for name in _XF:
        mods[name] = types.ModuleType(name)
        sys.modules[name] = mods[name]

    class Original:
        pass
    mods[_XF[-1]].FusedMLP = Original
    assert M.install_shims() is True
    assert mods[_XF[-1]].FusedMLP is M.FusedMLP
    from xformers.components.feedforward import fused_mlp          # the reference's own lookup
    assert fused_mlp.FusedMLP is M.FusedMLP


def test_install_shims_does_nothing_without_xformers(saved_xformers):
    M = _mlp()
    for name in _XF:
        sys.modules[name] = None          # makes `import xformers...` raise ImportError
    assert M.install_shims() is False


def test_package_install_shims_leaves_fused_mlp_alone(saved_xformers):
    import gaussiananything_b200 as ga
    mod = types.ModuleType(_XF[-1])

    class Original:
        pass
    mod.FusedMLP = Original
    sys.modules[_XF[-1]] = mod
    saved = {k: sys.modules.get(k) for k in ("diff_surfel_rasterization", "transport", "transport.transport",
                                            "transport.path", "transport.integrators")}
    try:
        ga.install_shims()
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    assert mod.FusedMLP is Original
    assert ga.mlp.FusedMLP is _mlp().FusedMLP


# ---- host-only argument check of the C library ---------------------------------------------------------------------

def test_linear_grad_validate_rules():
    """ga_linear_grad_validate makes no CUDA call: fake, never dereferenced addresses.  Every rule of the header, one
    at a time, from an accepted call of each op."""
    from gaussiananything_b200 import _lib
    L = _lib.lib()
    A, B, AUX, OUT, WS = 0x100000, 0x200000, 0x300000, 0x400000, 0x500000
    M, N, K = 3072, 256, 1024
    ws_w = L.ga_linear_wgrad_workspace_bytes(M, N, K)
    ws_b = L.ga_linear_bias_grad_workspace_bytes(M, N)
    assert ws_w > 0 and ws_b > 0

    base = {
        _lib.LINEAR_FC1: dict(a=A, b=B, aux=AUX, out=OUT, f32=0, bn=128, ws=None, wsb=0),
        _lib.LINEAR_DGRAD: dict(a=A, b=B, aux=AUX, out=OUT, f32=0, bn=0, ws=None, wsb=0),
        _lib.LINEAR_WGRAD: dict(a=A, b=B, aux=None, out=OUT, f32=1, bn=0, ws=WS, wsb=ws_w),
        _lib.LINEAR_BGRAD: dict(a=A, b=None, aux=None, out=OUT, f32=1, bn=0, ws=WS, wsb=ws_b),
    }

    def rc(op, **kw):
        a = dict(base[op], M=M, N=N, K=K)
        a.update(kw)
        return L.ga_linear_grad_validate(op, a["a"], a["b"], a["aux"], a["out"], a["f32"], a["M"], a["N"], a["K"],
                                         a["bn"], a["ws"], a["wsb"])

    for op in base:
        assert rc(op) == 0, op
        big = dict(wsb=1 << 40) if op in (_lib.LINEAR_WGRAD, _lib.LINEAR_BGRAD) else {}
        assert rc(op, M=1) == 0 and rc(op, M=98304, **big) == 0 and rc(op, M=127) == 0, op
        for kw in (dict(a=None), dict(a=A + 8), dict(out=None), dict(out=OUT + 4), dict(M=0), dict(M=-1),
                   dict(N=0), dict(N=12), dict(N=4), dict(M=1 << 20, N=4096)):
            assert rc(op, **kw) == -1, (op, kw)
        if op != _lib.LINEAR_BGRAD:
            for kw in (dict(b=None), dict(b=B + 2), dict(K=0), dict(K=20), dict(N=8, K=1 << 28)):
                assert rc(op, **kw) == -1, (op, kw)
    FC1, DG, WG, BG = _lib.LINEAR_FC1, _lib.LINEAR_DGRAD, _lib.LINEAR_WGRAD, _lib.LINEAR_BGRAD
    # fc1: Z required; bf16 outputs; ga_gemm_bf16_tn's tile widths
    assert rc(FC1, aux=None) == -1 and rc(FC1, aux=AUX + 8) == -1 and rc(FC1, f32=1) == -1
    assert all(rc(FC1, bn=bn) == 0 for bn in (64, 128, 192, 256))
    assert rc(FC1, bn=96) == -1 and rc(FC1, bn=0) == -1
    # dgrad: Z optional; fp32 output only without Z
    assert rc(DG, aux=None) == 0 and rc(DG, aux=None, f32=1) == 0
    assert rc(DG, f32=1) == -1 and rc(DG, aux=AUX + 8) == -1 and rc(DG, aux=None, f32=2) == -1
    # wgrad / bias: fp32 output, a workspace large enough when one is needed
    for op, need in ((WG, ws_w), (BG, ws_b)):
        assert rc(op, f32=0) == -1 and rc(op, wsb=need - 1) == -1 and rc(op, ws=None) == -1 and rc(op, ws=WS + 8) == -1
        assert rc(op, wsb=need + 64) == 0
    assert rc(BG, K=0) == 0 and rc(BG, K=3) == 0                                    # K unused
    # one split or one chunk: no workspace at all
    assert L.ga_linear_wgrad_workspace_bytes(3072, 4096, 1024) == 0 and rc(WG, N=4096, ws=None, wsb=0) == 0
    assert L.ga_linear_bias_grad_workspace_bytes(256, N) == 0 and rc(BG, M=256, ws=None, wsb=0) == 0
    for op in (-1, 4):
        assert L.ga_linear_grad_validate(op, A, B, AUX, OUT, 0, M, N, K, 128, WS, 1 << 40) == -1


def test_wgrad_splits_depend_on_the_shapes_only():
    from gaussiananything_b200 import _lib
    L = _lib.lib()
    S = L.ga_linear_wgrad_splits
    assert S(3072, 4096, 1024) == 1 and S(3072, 1024, 4096) == 1                     # DiT-L: 256 tiles already
    assert S(768, 256, 1024) > 1 and S(768, 1024, 256) > 1                          # SRT: 16 tiles
    assert S(64, 256, 1024) == 1 and S(1, 8, 8) == 1                                # too few rows to split
    for M, N, K in ((768, 256, 1024), (98304, 768, 3072), (3072, 768, 3072)):
        s = S(M, N, K)
        assert 1 <= s <= 32 and 2 * s <= max(2, (M + 63) // 64)
        assert L.ga_linear_wgrad_workspace_bytes(M, N, K) == (s * N * K * 4 if s > 1 else 0)
