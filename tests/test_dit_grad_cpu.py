"""CPU checks of the trainable DiT block (include/ga_b200.h Part 14, gaussiananything_b200/dit_grad.py): the
references against autograd, every refusal of the module and the function, the host-only argument checks of the C
library, and the block's state dict and forward signature against the reference's."""
import inspect
import json
import os

import pytest
import torch

from tests import dit_grad_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _block(D=128, H=2, Dc=64, seed=0):
    from gaussiananything_b200 import dit
    torch.manual_seed(seed)
    b = dit.ImageCondDiTBlockPixelArtRMSNormClayLRM(D, H, Dc)
    with torch.no_grad():
        for name, p in b.named_parameters():
            if name.endswith("bias") or "norm" in name:
                p.add_(0.1 * torch.randn_like(p))
    return b


def _case(B=2, N=5, M=3, D=128, Dc=64, seed=1):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, N, D, generator=g), 0.3 * torch.randn(B, 6 * D, generator=g),
            torch.randn(B, M, Dc, generator=g), torch.randn(B, N, D, generator=g))


def test_restated_block_is_the_oracle():
    """With its roundings off the emulation's code is the oracle's block_forward: y and every gradient agree (to the
    oracle's RMSNorm, which takes the variance in fp32 whatever the input's dtype)."""
    b = _block()
    sd = {k: v.detach() for k, v in b.state_dict().items()}
    x, t, c, dy = _case()
    ref = R.block(sd, x, t, c, 2, dy)
    res = R.block(sd, x, t, c, 2, dy, restated=True)
    assert set(ref) == set(R.PARAMS) | {"y", "dx", "dt", "dctx"}
    for k in ref:
        assert R.rel_l2(res[k], ref[k]) < 1e-7, k


def test_fp64_reference_matches_finite_differences():
    """Central differences of the restated block (all fp64) against the autograd gradients."""
    b = _block(D=64, H=1, Dc=8)
    sd = {k: v.detach().double() for k, v in b.state_dict().items()}
    x, t, c, dy = _case(B=1, N=3, M=2, D=64, Dc=8)
    ref = R.block(sd, x, t, c, 1, dy, restated=True)
    eps = 1e-6
    for name, idx in (("dx", (0, 1, 3)), ("dt", (0, 70)), ("dctx", (0, 1, 5))):
        base = {"dx": x, "dt": t, "dctx": c}[name].double()
        e = torch.zeros_like(base)
        e[idx] = eps
        f = lambda d: R._block_emu(sd, *[(base + d) if n == name else v.double()
                                         for n, v in (("dx", x), ("dt", t), ("dctx", c))], 1, rounding=False)
        fd = float(((f(e) - f(-e)) * dy.double()).sum() / (2 * eps))
        assert abs(fd - float(ref[name][idx])) < 1e-6 * max(1.0, abs(fd)), name


def test_emulation_rounds_and_stays_close():
    b = _block()
    for p in b.parameters():
        p.data.copy_(R.bf16(p.data))
    sd = {k: v.detach() for k, v in b.state_dict().items()}
    x, t, c, dy = _case(N=40, M=17)
    ref = R.block(sd, x, t, c, 2, dy)
    emu = R.block(sd, x, t, c, 2, dy, emulate=True)
    for k in ref:
        d = R.rel_l2(emu[k], ref[k])
        assert 1e-5 < d < 3e-2, (k, d)


# ---- refusals -------------------------------------------------------------------------------------------------------

def test_cpu_tensors_raise():
    b = _block()
    x, t, c, _ = _case()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        b(x, t, c)
    from gaussiananything_b200 import dit_grad
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        dit_grad.block_forward(b, x.requires_grad_(), t, c)


def test_head_dim_other_than_64_raises():
    from gaussiananything_b200 import dit
    b = dit.ImageCondDiTBlockPixelArtRMSNormClayLRM(128, 4, 64)          # head_dim 32
    x, t, c, _ = _case()
    with pytest.raises(NotImplementedError, match="head_dim"):
        b(x, t, c)


def test_rope_raises_and_caption_is_ignored_by_signature():
    b = _block()
    x, t, c, _ = _case()
    with pytest.raises(NotImplementedError, match="RoPE"):
        b(x, t, c, None, freqs_cis=torch.zeros(5, 32))


@pytest.mark.parametrize("what", ["x_rank", "x_width", "t_size", "ctx_batch", "ctx_width", "x_dtype", "t_type"])
def test_shape_and_type_refusals(what):
    b = _block()
    x, t, c, _ = _case()
    bad = dict(x_rank=(x[0], t, c), x_width=(x[..., :64], t, c), t_size=(x, t[:, :-1], c), ctx_batch=(x, t, c[:1]),
               ctx_width=(x, t, c[..., :32]), x_dtype=(x.double(), t, c), t_type=(x, 1.0, c))[what]
    exc = TypeError if what in ("x_dtype", "t_type") else ValueError
    with pytest.raises(exc):
        b(*bad)


def test_state_dict_and_forward_signature_match_the_reference():
    keys = json.load(open(os.path.join(ROOT, "tests", "golden", "dit_state_dict_keys.json")))["DiT-PixArt-PCD-CLAY-L"]
    want = {k[len("blocks.0."):]: tuple(v) for k, v in keys.items() if k.startswith("blocks.0.")}
    from gaussiananything_b200 import dit
    b = dit.ImageCondDiTBlockPixelArtRMSNormClayLRM(1024, 16, 1024)
    assert {k: tuple(v.shape) for k, v in b.state_dict().items()} == want
    # dit/dit_models_xformers.py:765: forward(self, x, t, dino_spatial_token, clip_caption_token=None,
    #                                         freqs_cis=None, **kwargs)
    sig = inspect.signature(b.forward)
    assert [(p.name, p.kind, p.default) for p in sig.parameters.values()] == [
        ("x", inspect.Parameter.POSITIONAL_OR_KEYWORD, inspect.Parameter.empty),
        ("t", inspect.Parameter.POSITIONAL_OR_KEYWORD, inspect.Parameter.empty),
        ("dino_spatial_token", inspect.Parameter.POSITIONAL_OR_KEYWORD, inspect.Parameter.empty),
        ("clip_caption_token", inspect.Parameter.POSITIONAL_OR_KEYWORD, None),
        ("freqs_cis", inspect.Parameter.POSITIONAL_OR_KEYWORD, None),
        ("kwargs", inspect.Parameter.VAR_KEYWORD, inspect.Parameter.empty)]
    from gaussiananything_b200 import dit_grad
    names = [n for n, _ in b.named_parameters() if not n.startswith("attention_y_norm")]
    assert len(dit_grad.block_parameters(b)) == 21 == len(names)
    by_id = {id(p): n for n, p in b.named_parameters()}
    assert tuple(by_id[id(p)] for p in dit_grad.block_parameters(b)) == R.PARAMS


def test_the_model_stays_inference_only():
    from gaussiananything_b200 import dit
    m = dit.DiT_I23D_PCD_PixelArt_noclip(input_size=32, num_classes=0, learn_sigma=False, in_channels=3,
                                         context_dim=64, roll_out=True, depth=1, hidden_size=128, num_heads=2)
    with pytest.raises(RuntimeError):
        m(torch.randn(1, 4, 3), torch.rand(1), {"img_crossattn": torch.randn(1, 3, 64), "img_vector": torch.randn(1, 64)})


# ---- host-only argument checks of the C library ---------------------------------------------------------------------

def _L():
    from gaussiananything_b200 import _lib
    return _lib.lib()


def test_partial_counts_depend_on_the_shapes_only():
    L = _L()
    assert L.ga_dit_grad_partials(3072, 768) == 4 * 24
    assert L.ga_dit_grad_partials(4 * 65, 65) == 4 * 3 and L.ga_dit_grad_partials(1, 1) == 1
    assert L.ga_dit_grad_partials(5476, 5476) == 172
    assert L.ga_dit_grad_partials(10, 3) == 0 and L.ga_dit_grad_partials(0, 1) == 0


def test_rmsnorm_bwd_validate_rules():
    L = _L()
    A = dict(dh=0x100000, x=0x200000, w=0x300000, scale=0x400000, mod_ld=6144, dx_in=0x500000, dx_out=0x600000,
             pdw=0x700000, psh=0x800000, psc=0x900000, pld=6144, rpb=768, R=3072, D=1024)

    def rc(**kw):
        a = dict(A, **kw)
        return L.ga_dit_rmsnorm_bwd_validate(a["dh"], a["x"], a["w"], a["scale"], a["mod_ld"], a["dx_in"],
                                             a["dx_out"], a["pdw"], a["psh"], a["psc"], a["pld"], a["rpb"], a["R"],
                                             a["D"])
    assert rc() == 0 and rc(dx_in=None) == 0 and rc(dx_in=None, dx_out=None) == 0
    assert rc(scale=None, psh=None, psc=None) == 0 and rc(D=4, mod_ld=4, pld=4) == 0 and rc(R=1, rpb=1) == 0
    for kw in (dict(dh=None), dict(x=None), dict(w=None), dict(pdw=None), dict(dh=0x100004), dict(w=0x300008),
               dict(dx_out=None), dict(dx_in=0x500004), dict(dx_out=0x600008), dict(scale=0x400004),
               dict(mod_ld=1020), dict(mod_ld=6146), dict(psh=None), dict(psc=None), dict(pld=1000),
               dict(scale=None), dict(scale=None, psh=None), dict(R=3000), dict(rpb=0), dict(R=0), dict(D=1028),
               dict(D=1022), dict(D=0), dict(R=1 << 21, rpb=1 << 21)):
        assert rc(**kw) == -1, kw


def test_gate_validate_rules():
    L = _L()
    A = dict(dy=0x100000, a=0x200000, gate=0x300000, gld=6144, da=0x400000, part=0x500000, pld=6144, rpb=768,
             R=3072, D=1024)

    def rc(**kw):
        a = dict(A, **kw)
        return L.ga_dit_gate_bwd_validate(a["dy"], a["a"], a["gate"], a["gld"], a["da"], a["part"], a["pld"],
                                          a["rpb"], a["R"], a["D"])
    assert rc() == 0 and rc(da=0x400008) == 0
    for kw in (dict(dy=None), dict(a=None), dict(gate=None), dict(da=None), dict(part=None), dict(da=0x400004),
               dict(gate=0x300004), dict(gld=1000), dict(pld=6146), dict(R=3071), dict(D=2048)):
        assert rc(**kw) == -1, kw
    G = dict(x=0x100000, a=0x200000, gate=0x300000, gld=6144, xo=0x400000, w=0x500000, sh=0x600000, sc=0x700000,
             mld=6144, h=0x800000, rpb=768, R=3072, D=1024)

    def rg(**kw):
        a = dict(G, **kw)
        return L.ga_dit_gate_residual_validate(a["x"], a["a"], a["gate"], a["gld"], a["xo"], a["w"], a["sh"],
                                               a["sc"], a["mld"], a["h"], a["rpb"], a["R"], a["D"])
    assert rg() == 0 and rg(gate=None, gld=0) == 0 and rg(sh=None, sc=None, mld=0) == 0
    assert rg(w=None, sh=None, sc=None, h=None) == 0
    for kw in (dict(x=None), dict(a=None), dict(xo=None), dict(x=0x100008), dict(gate=0x300004), dict(gld=1020),
               dict(w=None), dict(h=None), dict(h=0x800004), dict(sh=None), dict(sc=None), dict(mld=1000),
               dict(w=None, sh=None, sc=None), dict(w=0x500004), dict(rpb=5), dict(D=6)):
        assert rg(**kw) == -1, kw


def test_qk_norm_and_reduce_validate_rules():
    L = _L()
    A = dict(bwd=1, src=0x100000, ld_in=3072, d=0x200000, ld_d=3072, out=0x300000, ld_out=3072, w0=0x400000,
             w1=0x500000, part=0x600000, rows=3072, heads=16, parts=2)

    def rc(**kw):
        a = dict(A, **kw)
        return L.ga_dit_qk_norm_validate(a["bwd"], a["src"], a["ld_in"], a["d"], a["ld_d"], a["out"], a["ld_out"],
                                         a["w0"], a["w1"], a["part"], a["rows"], a["heads"], a["parts"])
    assert rc() == 0 and rc(bwd=0, d=None, part=None) == 0 and rc(parts=1, w1=None, ld_in=1024, ld_d=1024,
                                                                    ld_out=1024) == 0
    for kw in (dict(bwd=2), dict(src=None), dict(out=None), dict(w0=None), dict(w1=None), dict(parts=1),
               dict(parts=3), dict(rows=0), dict(heads=0), dict(ld_in=2040), dict(ld_in=3076), dict(ld_out=2040),
               dict(ld_d=2040), dict(d=None), dict(part=None), dict(src=0x100008), dict(d=0x200008),
               dict(out=0x300008), dict(w0=0x400004), dict(part=0x600004), dict(bwd=0), dict(bwd=0, d=None)):
        assert rc(**kw) == -1, kw
    assert L.ga_dit_grad_reduce_validate(0x100000, 0x200000, 4, 24, 6144) == 0
    for a in ((None, 0x200000, 1, 1, 1), (0x100000, None, 1, 1, 1), (0x100000, 0x200000, 0, 1, 1),
              (0x100000, 0x200000, 1, 0, 1), (0x100000, 0x200000, 1, 1, 0)):
        assert L.ga_dit_grad_reduce_validate(*a) == -1, a
