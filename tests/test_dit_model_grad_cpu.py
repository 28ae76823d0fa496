"""CPU checks of the trainable image-to-3D DiT (include/ga_b200.h Part 15, gaussiananything_b200/dit_grad.py
model_forward): the fp64 restatement against the oracle on the reference's goldens, finite differences of the stem and
head, every refusal of model_forward and the host-only argument checks of the new C entry points."""
import os

import pytest
import torch

from tests import dit_model_grad_ref as MR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


@pytest.mark.parametrize("name", ["dit_stage1_small", "dit_stage2_small", "dit_stage2_concat_small"])
def test_restatement_is_the_oracle_on_the_goldens(name):
    from oracle import dit_oracle as do
    g = do.load_golden(os.path.join(GOLD, name + ".npz"))
    c = g["cfg"]
    y = MR.forward(g["sd"], g["x"], g["t"], g["ctx"], c["heads"], c["depth"])
    want = do.forward(g["sd"], g["x"], g["t"], g["ctx"], c["heads"], c["depth"])
    assert MR.rel_l2(y, want) < 1e-5
    assert MR.rel_l2(y, g["y"]) < 1e-5                    # the reference's own output


def _small_model_sd(pe=True, seed=0, D=64, Dc=16, Cin=4, Cout=5):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: 0.3 * torch.randn(*s, generator=g, dtype=torch.float64)
    P = {"t_embedder.mlp.0.weight": r(D, 256), "t_embedder.mlp.0.bias": r(D), "t_embedder.mlp.2.weight": r(D, D),
         "t_embedder.mlp.2.bias": r(D), "pooled_vec_embedder.0.weight": 1 + r(Dc),
         "pooled_vec_embedder.0.bias": r(Dc), "pooled_vec_embedder.1.weight": r(D, Dc),
         "pooled_vec_embedder.1.bias": r(D), "adaLN_modulation.1.weight": r(6 * D, D),
         "adaLN_modulation.1.bias": r(6 * D), "x_embedder.fc1.weight": r(D, Cin + (0 if pe else 3)),
         "x_embedder.fc1.bias": r(D), "x_embedder.fc2.weight": r(D, D), "x_embedder.fc2.bias": r(D),
         "final_layer.scale_shift_table": r(2, D), "final_layer.linear.weight": r(Cout, D),
         "final_layer.linear.bias": r(Cout)}
    if pe:
        P["xyz_pos_embed.xyz_projection.weight"], P["xyz_pos_embed.xyz_projection.bias"] = r(D, 63), r(D)
    return P


@pytest.mark.parametrize("pe", [True, False])
def test_stem_and_head_match_finite_differences(pe):
    """Central differences (fp64) of sum(dxres xres) + sum(dt0 t0) + sum(dtemb temb) and of sum(dy head) against the
    autograd gradients of the restated stem and head, for a few entries of every input and parameter."""
    P = _small_model_sd(pe)
    g = torch.Generator().manual_seed(3)
    B, N, D, Dc, Cin = 2, 3, 64, 16, 4
    x, vec, xyz = (torch.randn(*s, generator=g, dtype=torch.float64) for s in ((B, N, Cin), (B, Dc), (B, N, 3)))
    t = torch.tensor([0.3, 0.8], dtype=torch.float64)
    gx, gt0, gte = (torch.randn(*s, generator=g, dtype=torch.float64) for s in ((B, N, D), (B, 6 * D), (B, D)))
    h, dyh = torch.randn(B, N, D, generator=g, dtype=torch.float64), torch.randn(B, N, 5, generator=g,
                                                                                 dtype=torch.float64)

    def stem_loss(Q, xx, vv):
        a, b, c = MR.stem(Q, xx, t, vv, xyz)
        return (a * gx).sum() + (b * gt0).sum() + (c * gte).sum()

    def head_loss(Q, hh, te):
        return (MR.head(Q, hh, te) * dyh).sum()

    leaves = {k: v.clone().requires_grad_(True) for k, v in P.items()}
    xs = [v.clone().requires_grad_(True) for v in (x, vec, h, gte)]
    (stem_loss(leaves, xs[0], xs[1]) + head_loss(leaves, xs[2], xs[3])).backward()
    eps = 1e-6
    checks = [("x", xs[0], (0, 1, 2)), ("vec", xs[1], (1, 7)), ("h", xs[2], (1, 2, 30)), ("temb", xs[3], (0, 9))]
    checks += [(k, leaves[k], tuple(int(i) % s for i, s in zip((5, 77, 3), v.shape))) for k, v in P.items()]
    for name, leaf, idx in checks:
        def f(d):
            Q = {k: (v + d if k == name else v) for k, v in P.items()}
            args = {n: (v + d if n == name else v) for n, v in (("x", x), ("vec", vec), ("h", h), ("temb", gte))}
            return float(stem_loss(Q, args["x"], args["vec"]) + head_loss(Q, args["h"], args["temb"]))
        e = torch.zeros_like(leaf)
        e[idx] = eps
        fd = (f(e) - f(-e)) / (2 * eps)
        assert abs(fd - float(leaf.grad[idx])) < 1e-6 * max(1.0, abs(fd)), (name, idx, fd, float(leaf.grad[idx]))


def test_emulation_rounds_and_stays_close():
    from oracle import dit_oracle as do
    g = do.load_golden(os.path.join(GOLD, "dit_stage2_small.npz"))
    c = g["cfg"]
    dy = torch.randn(g["y"].shape, generator=torch.Generator().manual_seed(0))
    ref = MR.model(g["sd"], g["x"], g["t"], g["ctx"], c["heads"], c["depth"], dy)
    emu = MR.model(g["sd"], g["x"], g["t"], g["ctx"], c["heads"], c["depth"], dy, emulate=True)
    assert set(ref) == {"y", "dx", "dctx", "dvec"} | set(MR.param_names(g["sd"], c["depth"]))
    for k in ref:
        d = MR.rel_l2(emu[k], ref[k])
        assert d < 5e-2, (k, d)
    assert MR.rel_l2(emu["x_embedder.fc2.weight"], ref["x_embedder.fc2.weight"]) > 1e-5


# ---- refusals -------------------------------------------------------------------------------------------------------

def _model(stage=1, pe=True, Cin=3, learn_sigma=False, depth=1):
    from gaussiananything_b200 import dit
    kw = dict(input_size=32, num_classes=0, learn_sigma=learn_sigma, in_channels=Cin, context_dim=64, roll_out=True,
              depth=depth, hidden_size=128, num_heads=2)
    if stage == 1:
        return dit.DiT_I23D_PCD_PixelArt_noclip(**kw)
    return dit.DiT_I23D_PCD_PixelArt_noclip_clay_stage2(use_pe_cond=pe, **kw)


def _inputs(B=2, N=5, M=3, Cin=3, stage2=False):
    g = torch.Generator().manual_seed(0)
    ctx = {"img_crossattn": torch.randn(B, M, 64, generator=g), "img_vector": torch.randn(B, 64, generator=g)}
    if stage2:
        ctx["fps-xyz"] = torch.randn(B, N, 3, generator=g)
    return torch.randn(B, N, Cin, generator=g), torch.rand(B, generator=g), ctx


def test_cpu_tensors_raise():
    from gaussiananything_b200 import dit_grad
    m = _model()
    x, t, ctx = _inputs()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        dit_grad.model_forward(m, x.requires_grad_(), t, ctx)


def test_text_to_3d_model_raises():
    from gaussiananything_b200 import dit_grad, dit_t23d
    m = dit_t23d.DiT_PCD_PixelArt(input_size=32, num_classes=0, learn_sigma=False, in_channels=3, context_dim=64,
                                  roll_out=True, depth=1, hidden_size=128, num_heads=2, patch_size=1)
    x, t, ctx = _inputs()
    with pytest.raises(NotImplementedError, match="text-to-3D"):
        dit_grad.model_forward(m, x, t, ctx)


@pytest.mark.parametrize("which", ["timesteps", "fps-xyz"])
def test_constants_requiring_grad_raise(which):
    from gaussiananything_b200 import dit_grad
    m = _model(stage=2)
    x, t, ctx = _inputs(stage2=True)
    if which == "timesteps":
        t.requires_grad_(True)
    else:
        ctx["fps-xyz"].requires_grad_(True)
    with pytest.raises(ValueError, match="constant"):
        dit_grad.model_forward(m, x, t, ctx)


def test_wide_output_raises():
    from gaussiananything_b200 import dit_grad
    m = _model(Cin=9, learn_sigma=True)                            # out_channels 18 > 16
    x, t, ctx = _inputs(Cin=9)
    with pytest.raises(NotImplementedError, match="out_channels 18"):
        dit_grad.model_forward(m, x, t, ctx)


def test_wide_embedder_input_raises():
    from gaussiananything_b200 import dit_grad
    m = _model(stage=2, pe=False, Cin=14)                          # 14 + 3 xyz > 16
    x, t, ctx = _inputs(Cin=14, stage2=True)
    with pytest.raises(NotImplementedError, match="17 inputs"):
        dit_grad.model_forward(m, x, t, ctx)


@pytest.mark.parametrize("what", ["x_width", "t_size", "vec_size", "xyz_missing", "xyz_size", "t_none", "x_dtype",
                                  "ctx_type"])
def test_shape_and_type_refusals(what):
    from gaussiananything_b200 import dit_grad
    m = _model(stage=2)
    x, t, ctx = _inputs(stage2=True)
    drop = lambda k: {a: b for a, b in ctx.items() if a != k}
    bad = dict(x_width=(x[..., :2], t, ctx), t_size=(x, torch.rand(3), ctx),
               vec_size=(x, t, dict(ctx, img_vector=ctx["img_vector"][:, :32])),
               xyz_missing=(x, t, drop("fps-xyz")), xyz_size=(x, t, dict(ctx, **{"fps-xyz": ctx["fps-xyz"][:, :2]})),
               t_none=(x, None, ctx), x_dtype=(x.double(), t, ctx), ctx_type=(x, t, [ctx]))[what]
    exc = TypeError if what in ("t_none", "x_dtype") else ValueError
    with pytest.raises(exc):
        dit_grad.model_forward(m, *bad)


def test_rope_raises():
    from gaussiananything_b200 import dit_grad
    m = _model()
    m.freqs_cis = torch.zeros(5, 32)
    x, t, ctx = _inputs()
    with pytest.raises(NotImplementedError, match="RoPE"):
        dit_grad.model_forward(m, x, t, ctx)


def test_stem_and_head_parameters_are_the_state_dict_names():
    from gaussiananything_b200 import dit_grad
    for m, pe in ((_model(), False), (_model(stage=2, pe=True), True), (_model(stage=2, pe=False), False)):
        by_id = {id(p): n for n, p in m.named_parameters()}
        assert tuple(by_id[id(p)] for p in dit_grad.stem_parameters(m)) == MR.STEM + (MR.PE if pe else ())
        assert tuple(by_id[id(p)] for p in dit_grad.head_parameters(m)) == MR.HEAD


# ---- host-only argument checks of the C library ---------------------------------------------------------------------

def _L():
    from gaussiananything_b200 import _lib
    return _lib.lib()


def test_final_layer_bwd_validate_rules():
    L = _L()
    A = dict(x=0x100000, mod=0x200000, W=0x300000, dy=0x400000, dx=0x500000, pm=0x600000, pw=0x700000, pb=0x800000,
             rpb=768, R=3072, D=1024, C=16)

    def rc(**kw):
        a = dict(A, **kw)
        return L.ga_dit_final_layer_bwd_validate(a["x"], a["mod"], a["W"], a["dy"], a["dx"], a["pm"], a["pw"],
                                                 a["pb"], a["rpb"], a["R"], a["D"], a["C"])
    assert rc() == 0 and rc(dx=None) == 0 and rc(pm=None) == 0 and rc(pw=None, pb=None) == 0
    assert rc(C=1) == 0 and rc(D=4) == 0 and rc(R=1, rpb=1) == 0 and rc(dy=0x400004, pb=0x800004) == 0
    for kw in (dict(x=None), dict(mod=None), dict(W=None), dict(dy=None), dict(pw=None), dict(pb=None),
               dict(x=0x100004), dict(mod=0x200008), dict(W=0x300004), dict(dx=0x500004), dict(pm=0x600008),
               dict(pw=0x700004), dict(dy=0x400002), dict(pb=0x800002), dict(C=0), dict(C=17), dict(D=1028),
               dict(D=6), dict(D=0), dict(R=3000), dict(rpb=0), dict(R=0), dict(R=1 << 21, rpb=1 << 21)):
        assert rc(**kw) == -1, kw


def test_embed_fc1_bwd_validate_rules():
    L = _L()
    A = dict(x=0x100000, Cx=10, x2=0x200000, C2=3, W=0x300000, b=0x400000, de=0x500000, pw=0x600000, pb=0x700000,
             dx=0x800000, R=3072, D=1024)

    def rc(**kw):
        a = dict(A, **kw)
        return L.ga_dit_embed_fc1_bwd_validate(a["x"], a["Cx"], a["x2"], a["C2"], a["W"], a["b"], a["de"], a["pw"],
                                               a["pb"], a["dx"], a["R"], a["D"])
    assert rc() == 0 and rc(dx=None) == 0 and rc(C2=0, x2=None) == 0 and rc(Cx=13) == 0 and rc(D=1, R=1) == 0
    for kw in (dict(x=None), dict(W=None), dict(b=None), dict(de=None), dict(pw=None), dict(pb=None),
               dict(x2=None), dict(C2=0), dict(Cx=0), dict(Cx=14), dict(C2=-1, x2=None), dict(D=1025), dict(D=0),
               dict(R=0), dict(x=0x100002), dict(de=0x500001), dict(dx=0x800002), dict(R=1 << 21)):
        assert rc(**kw) == -1, kw


def test_linear_small_bwd_validate_rules():
    L = _L()
    A = dict(x=0x100000, act=1, W=0x200000, dy=0x300000, dW=0x400000, db=0x500000, part=0x600000, dxin=0x700000,
             dx=0x700000, rows=4, N=6144, K=1024)

    def rc(**kw):
        a = dict(A, **kw)
        return L.ga_dit_linear_small_bwd_validate(a["x"], a["act"], a["W"], a["dy"], a["dW"], a["db"], a["part"],
                                                  a["dxin"], a["dx"], a["rows"], a["N"], a["K"])
    assert rc() == 0 and rc(act=0) == 0 and rc(dW=None, db=None) == 0 and rc(dxin=None) == 0
    assert rc(dx=None, part=None, dxin=None) == 0 and rc(rows=20) == 0 and rc(N=1, K=4) == 0
    assert rc(dy=0x300004, db=0x500004, dx=0x700004, dxin=0x700004) == 0
    for kw in (dict(x=None), dict(W=None), dict(dy=None), dict(part=None), dict(dx=None), dict(dx=None, part=None),
               dict(act=2), dict(rows=0), dict(N=0), dict(K=0), dict(K=6), dict(K=2), dict(x=0x100004),
               dict(W=0x200008), dict(dW=0x400004), dict(part=0x600004), dict(dy=0x300002), dict(dx=0x700002),
               dict(N=1 << 20, K=4096), dict(rows=100000)):
        assert rc(**kw) == -1, kw


def test_layernorm_rows_bwd_validate_rules():
    L = _L()
    A = dict(x=0x100000, w=0x200000, dy=0x300000, dx=0x400000, dw=0x500000, db=0x600000, R=4, D=1024)

    def rc(**kw):
        a = dict(A, **kw)
        return L.ga_dit_layernorm_rows_bwd_validate(a["x"], a["w"], a["dy"], a["dx"], a["dw"], a["db"], a["R"],
                                                    a["D"])
    assert rc() == 0 and rc(dx=None, dw=None, db=None) == 0 and rc(D=4) == 0 and rc(R=1000) == 0
    for kw in (dict(x=None), dict(w=None), dict(dy=None), dict(x=0x100004), dict(dx=0x400008), dict(dw=0x500004),
               dict(db=0x600004), dict(R=0), dict(D=0), dict(D=1028), dict(D=6)):
        assert rc(**kw) == -1, kw
