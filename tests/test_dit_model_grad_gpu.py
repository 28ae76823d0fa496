"""GPU checks of the trainable image-to-3D DiT (include/ga_b200.h Part 15, gaussiananything_b200/dit_grad.py
model_forward): each new kernel element by element against fp64, model_forward without grad against the inference
engine, every gradient of stage 1 and both stage-2 variants against fp64 within 1.5 times the bf16 emulation's
distance, repeatable bits, skipped GEMMs under frozen blocks or a frozen stem, the in-place and double-backward
errors, and a flow-matching AdamW run under bf16 autocast."""
import functools
import math
import os

import pytest
import torch

from tests import dit_model_grad_ref as MR

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NAN = float("nan")


def _L():
    from gaussiananything_b200 import _lib
    return _lib.lib()


def _st():
    import ctypes as C
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    import ctypes as C
    return C.c_void_p(t.data_ptr() if t is not None else 0)


def _close(got, ref, rtol, what):
    """every element within rtol of the row's largest |ref| plus rtol |ref| (NaN never is)"""
    ref = ref.double()
    err = (got.double() - ref).abs()
    scale = ref.abs().amax(dim=-1, keepdim=True).clamp_min(1e-30)
    ok = err <= rtol * (scale + ref.abs())
    assert bool(ok.all()), "%s: %d bad, worst err %.3e" % (what, int((~ok).sum()), float(err.max()))


def _reduce(part, groups, cols):
    out = torch.full((groups, cols), NAN, device=DEV)
    assert _L().ga_dit_grad_reduce(_p(part), _p(out), groups, part.numel() // (groups * cols), cols, _st()) == 0
    return out


# ---- kernels ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("B,N,D,Cout", [(1, 1, 64, 3), (4, 65, 1024, 10), (20, 33, 256, 16), (4, 32, 128, 3)])
def test_final_layer_bwd_kernel(B, N, D, Cout):
    L = _L()
    g = torch.Generator(device=DEV).manual_seed(N)
    R = B * N
    x = 2 * torch.randn(R, D, device=DEV, generator=g) + 0.5
    mod = 0.3 * torch.randn(B, 2 * D, device=DEV, generator=g)
    Wbuf = torch.full((16, D), NAN, device=DEV)                        # rows past Cout must not be read
    Wbuf[:Cout] = torch.randn(Cout, D, device=DEV, generator=g) / math.sqrt(D)
    dy = torch.randn(R, Cout, device=DEV, generator=g)
    P = L.ga_dit_grad_partials(R, N)
    dx = torch.full((R, D), NAN, device=DEV)
    pmod, pw, pb = (torch.full(s, NAN, device=DEV) for s in ((P, 2 * D), (P, Cout * D), (P, Cout)))
    assert L.ga_dit_final_layer_bwd(_p(x), _p(mod), _p(Wbuf), _p(dy), _p(dx), _p(pmod), _p(pw), _p(pb), N, R, D, Cout,
                                    1e-6, _st()) == 0
    xd, md, Wd, gd = x.double(), mod.double(), Wbuf[:Cout].double(), dy.double()
    mu = xd.mean(-1, keepdim=True)
    rs = torch.rsqrt((xd - mu).pow(2).mean(-1, keepdim=True) + 1e-6)
    n = (xd - mu) * rs
    sh, sc = md[:, :D].repeat_interleave(N, 0), md[:, D:].repeat_interleave(N, 0)
    dh = gd @ Wd
    dn = dh * (1 + sc)
    _close(dx, rs * (dn - dn.mean(-1, keepdim=True) - n * (dn * n).mean(-1, keepdim=True)), 1e-5, "dx")
    dmod = _reduce(pmod, B, 2 * D)
    _close(dmod[:, :D], dh.view(B, N, D).sum(1), 1e-5, "dshift")
    _close(dmod[:, D:], (dh * n).view(B, N, D).sum(1), 1e-5, "dscale")
    h = n * (1 + sc) + sh
    _close(_reduce(pw, 1, Cout * D).view(Cout, D), gd.t() @ h, 1e-5, "dW")
    _close(_reduce(pb, 1, Cout)[0], gd.sum(0), 1e-5, "db")
    # each output may be NULL: the others come out the same
    want = [t.clone() for t in (dx, pmod, pw, pb)]
    for t in (dx, pmod, pw, pb):
        t.fill_(NAN)
    assert L.ga_dit_final_layer_bwd(_p(x), _p(mod), _p(Wbuf), _p(dy), None, None, _p(pw), _p(pb), N, R, D, Cout,
                                    1e-6, _st()) == 0
    assert torch.equal(pw, want[2]) and torch.equal(pb, want[3])
    assert bool(torch.isnan(dx).all()) and bool(torch.isnan(pmod).all())
    assert L.ga_dit_final_layer_bwd(_p(x), _p(mod), _p(Wbuf), _p(dy), _p(dx), _p(pmod), None, None, N, R, D, Cout,
                                    1e-6, _st()) == 0
    assert torch.equal(dx, want[0]) and torch.equal(pmod, want[1])


@pytest.mark.parametrize("R,D,Cx,C2", [(1, 64, 3, 0), (4 * 65, 1024, 10, 3), (20 * 33, 256, 13, 3), (96, 128, 16, 0)])
def test_embed_fc1_bwd_kernel(R, D, Cx, C2):
    L = _L()
    g = torch.Generator(device=DEV).manual_seed(R)
    K = Cx + C2
    xin = torch.randn(R, Cx, device=DEV, generator=g)
    xin2 = torch.randn(R, C2, device=DEV, generator=g) if C2 else None
    W1 = torch.randn(D, K, device=DEV, generator=g) / math.sqrt(K)
    b1 = 0.1 * torch.randn(D, device=DEV, generator=g)
    de1 = torch.randn(R, D, device=DEV, generator=g)
    P = L.ga_dit_grad_partials(R, R)
    pw, pb = torch.full((P, D * K), NAN, device=DEV), torch.full((P, D), NAN, device=DEV)
    dxin = torch.full((R, Cx), NAN, device=DEV)
    assert L.ga_dit_embed_fc1_bwd(_p(xin), Cx, _p(xin2), C2, _p(W1), _p(b1), _p(de1), _p(pw), _p(pb), _p(dxin), R, D,
                                  _st()) == 0
    inp = torch.cat([xin2, xin], -1).double() if C2 else xin.double()
    v = (inp @ W1.double().t() + b1.double()).requires_grad_(True)
    torch.nn.functional.gelu(v, approximate="tanh").backward(de1.double())
    dv = v.grad
    _close(dxin, dv @ W1.double()[:, C2:], 1e-5, "dxin")
    _close(_reduce(pw, 1, D * K).view(D, K), dv.t() @ inp, 1e-5, "dW1")
    _close(_reduce(pb, 1, D)[0], dv.sum(0), 1e-5, "db1")
    # without dxin: the weight partials come out the same
    want_w, want_b = pw.clone(), pb.clone()
    pw.fill_(NAN)
    pb.fill_(NAN)
    assert L.ga_dit_embed_fc1_bwd(_p(xin), Cx, _p(xin2), C2, _p(W1), _p(b1), _p(de1), _p(pw), _p(pb), None, R, D,
                                  _st()) == 0
    assert torch.equal(pw, want_w) and torch.equal(pb, want_b)


@pytest.mark.parametrize("B,N,K,act", [(1, 64, 256, 0), (4, 6144, 1024, 1), (20, 1024, 1024, 1), (20, 77, 20, 1),
                                       (8, 33, 64, 0)])
def test_linear_small_bwd_kernel(B, N, K, act):
    L = _L()
    g = torch.Generator(device=DEV).manual_seed(N + K)
    x = torch.randn(B, K, device=DEV, generator=g)
    W = torch.randn(N, K, device=DEV, generator=g) / math.sqrt(K)
    dy = torch.randn(B, N, device=DEV, generator=g)
    dxin = torch.randn(B, K, device=DEV, generator=g)
    dW, db, dx = (torch.full(s, NAN, device=DEV) for s in ((N, K), (N,), (B, K)))
    part = torch.full((L.ga_dit_grad_partials(N, N), B, K), NAN, device=DEV)
    assert L.ga_dit_linear_small_bwd(_p(x), act, _p(W), _p(dy), _p(dW), _p(db), _p(part), _p(dxin), _p(dx), B, N, K,
                                     _st()) == 0
    xd = x.double().requires_grad_(True)
    a = torch.nn.functional.silu(xd) if act else xd
    (a @ W.double().t()).backward(dy.double())
    _close(dW, dy.double().t() @ a.detach(), 1e-5, "dW")
    _close(db, dy.double().sum(0), 1e-5, "db")
    _close(dx, dxin.double() + xd.grad, 1e-5, "dx")
    # dx_in == dx (in place), no dW or db
    dx2 = dxin.clone()
    assert L.ga_dit_linear_small_bwd(_p(x), act, _p(W), _p(dy), None, None, _p(part), _p(dx2), _p(dx2), B, N, K,
                                     _st()) == 0
    assert torch.equal(dx2, dx)


@pytest.mark.parametrize("B,D", [(1, 64), (4, 1024), (20, 768)])
def test_layernorm_rows_bwd_kernel(B, D):
    L = _L()
    g = torch.Generator(device=DEV).manual_seed(D)
    x = 3 * torch.randn(B, D, device=DEV, generator=g) + 1
    w, b = 1 + 0.2 * torch.randn(D, device=DEV, generator=g), torch.randn(D, device=DEV, generator=g)
    dy = torch.randn(B, D, device=DEV, generator=g)
    dx, dw, db = (torch.full(s, NAN, device=DEV) for s in ((B, D), (D,), (D,)))
    assert L.ga_dit_layernorm_rows_bwd(_p(x), _p(w), _p(dy), _p(dx), _p(dw), _p(db), B, D, 1e-5, _st()) == 0
    xs = [v.double().requires_grad_(True) for v in (x, w, b)]
    torch.nn.functional.layer_norm(xs[0], (D,), xs[1], xs[2], 1e-5).backward(dy.double())
    _close(dx, xs[0].grad, 1e-5, "dx")
    _close(dw, xs[1].grad, 1e-5, "dw")
    _close(db, xs[2].grad, 1e-5, "db")


# ---- the model --------------------------------------------------------------------------------------------------------

def _model(stage, pe, D, H, Dc, Cin, depth, learn_sigma=False, seed=0):
    from gaussiananything_b200 import dit
    torch.manual_seed(seed)
    kw = dict(input_size=32, num_classes=0, learn_sigma=learn_sigma, in_channels=Cin, context_dim=Dc, roll_out=True,
              depth=depth, hidden_size=D, num_heads=H, patch_size=1, pooling_ctx_dim=768, use_clay_ca=True)
    m = (dit.DiT_I23D_PCD_PixelArt_noclip(**kw) if stage == 1
         else dit.DiT_I23D_PCD_PixelArt_noclip_clay_stage2(use_pe_cond=pe, **kw))
    m.randomize_zero_init_(seed=seed)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if name.endswith("bias") or "norm" in name or "scale_shift" in name:
                p.add_(0.1 * torch.randn_like(p))
            p.copy_(p.to(torch.bfloat16).float())              # the values the tensor cores multiply
    return m.to(DEV)


def _inputs(stage, B, N, M, Cin, Dc, seed=1):
    g = torch.Generator(device=DEV).manual_seed(seed)
    ctx = {"img_crossattn": torch.randn(B, M, Dc, device=DEV, generator=g),
           "img_vector": torch.randn(B, Dc, device=DEV, generator=g)}
    if stage == 2:
        ctx["fps-xyz"] = torch.rand(B, N, 3, device=DEV, generator=g) - 0.5
    return torch.randn(B, N, Cin, device=DEV, generator=g), torch.rand(B, device=DEV, generator=g), ctx


def _run(m, x, t, ctx, dy):
    from gaussiananything_b200 import dit_grad
    for p in m.parameters():
        p.grad = None
    xs = x.clone().requires_grad_(True)
    c = dict(ctx, img_crossattn=ctx["img_crossattn"].clone().requires_grad_(True),
             img_vector=ctx["img_vector"].clone().requires_grad_(True))
    y = dit_grad.model_forward(m, xs, t, c)
    y.backward(dy)
    got = dict(y=y.detach(), dx=xs.grad, dctx=c["img_crossattn"].grad, dvec=c["img_vector"].grad)
    got.update({n: p.grad for n, p in m.named_parameters()})
    return got


@pytest.mark.parametrize("stage,pe,B,N,M", [(1, False, 2, 24, 10), (1, False, 20, 33, 9), (2, True, 20, 16, 7),
                                            (2, False, 4, 20, 9)])
def test_no_grad_forward_matches_the_engine(stage, pe, B, N, M):
    from gaussiananything_b200 import dit_grad
    m = _model(stage, pe, 128, 2, 64, 10 if stage == 2 else 3, 2).eval()
    x, t, ctx = _inputs(stage, B, N, M, m.in_channels, 64)
    with torch.no_grad():
        # the engine's stem takes at most 16 rows (ga_linear_small): B = 20 runs it on two halves
        want = torch.cat([m(x[i:i + 10], t[i:i + 10], {k: v[i:i + 10] for k, v in ctx.items()})
                          for i in range(0, B, 10)])
        got = dit_grad.model_forward(m, x, t, ctx)
    assert got.dtype == torch.float32 and got.shape == want.shape
    assert MR.rel_l2(got, want) < 6e-3                      # the block's bar against the engine's per-block taps
    for p in m.parameters():
        p.requires_grad_(False)
    y = dit_grad.model_forward(m, x, t, ctx)                # nothing requires grad: nothing is recorded
    assert y.grad_fn is None and torch.equal(y, got)


SHAPES = [  # stage, use_pe_cond, B, N, M, D, H, Dc, Cin, depth, learn_sigma
    (1, False, 1, 1, 1, 128, 2, 64, 3, 1, False),
    (1, False, 20, 33, 9, 128, 2, 64, 4, 2, True),
    (2, True, 2, 40, 7, 64, 1, 32, 10, 1, False),
    (2, False, 3, 20, 5, 192, 3, 32, 13, 1, False),
    (1, False, 4, 768, 1369, 1024, 16, 1024, 3, 2, False),   # DiT-L width, depth 2
    (2, True, 4, 768, 1369, 1024, 16, 1024, 3, 2, False),
    (2, False, 4, 768, 1369, 1024, 16, 1024, 3, 2, False),
]


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("stage,pe,B,N,M,D,H,Dc,Cin,depth,ls", SHAPES)
def test_gradients_against_fp64(stage, pe, B, N, M, D, H, Dc, Cin, depth, ls):
    m = _model(stage, pe, D, H, Dc, Cin, depth, learn_sigma=ls)
    x, t, ctx = _inputs(stage, B, N, M, Cin, Dc)
    dy = torch.randn(B, N, m.out_channels, device=DEV, generator=torch.Generator(device=DEV).manual_seed(7))
    got = _run(m, x, t, ctx, dy)
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    ref = MR.model(sd, x, t, ctx, H, depth, dy)
    emu = MR.model(sd, x, t, ctx, H, depth, dy, emulate=True)
    worst = []
    for k in ref:
        assert got[k] is not None and bool(torch.isfinite(got[k]).all()), k
        if not bool(ref[k].any()):
            assert float(got[k].double().norm()) <= 1e-3 * float(ref["dx"].norm()), k
            continue
        e_got, e_emu = MR.rel_l2(got[k], ref[k]), MR.rel_l2(emu[k], ref[k])
        worst.append((e_got / max(e_emu, 1e-30), k, e_got, e_emu))
        # the blocks' q/k-norm weight gradients keep tests/test_dit_grad_gpu.py's bound and its reason.  At DiT-L width
        # inside the model (D 1024, H 16, N 768, M 1369, depth 2, stage 1) the self-attention's measured 29.7 times
        # the emulation's distance (blocks.1 attn.q_norm.weight: 1.76e-1 against 5.9e-3).  block_forward alone, fed
        # this model's block-1 input, t0, context and output gradient, gives the same 35-38 times, and still 27-29
        # times with t0 swapped for the block test's 0.3 randn (the model's t0 has an rms of 0.26), so the loss is
        # the block backward's on this model's residual stream, not the stem's or the head's
        # (profiles/dit_train_h100.md).  Every other gradient of that shape stays within 1.5
        bound = 1.5
        if k.endswith(("q_norm.weight", "k_norm.weight")):
            bound = 40.0 if D == 1024 else 2.5
        assert e_got <= bound * e_emu + 2.0 ** -16, (k, e_got, e_emu)
    print("shape %s: worst ratio to the emulation %.2f (%s: %.2e vs %.2e)" % ((stage, pe, B, N, M, D), *max(worst)))
    for name in ("attention_y_norm.weight", "clip_spatial_proj.y_proj.fc1.weight", "cap_embedder.1.weight"):
        assert got[name] is None, name


def test_same_bits_on_repeated_calls():
    m = _model(2, True, 128, 2, 64, 10, 2)
    x, t, ctx = _inputs(2, 3, 40, 9, 10, 64)
    dy = torch.randn(3, 40, 10, device=DEV)
    a, b = _run(m, x, t, ctx, dy), _run(m, x, t, ctx, dy)
    for k in a:
        assert (a[k] is None and b[k] is None) or torch.equal(a[k], b[k]), k


@pytest.mark.parametrize("frozen", ["blocks", "stem"])
def test_frozen_parts_skip_their_gemms(frozen, monkeypatch):
    from gaussiananything_b200 import dit_grad
    m = _model(2, True, 128, 2, 64, 10, 2)
    x, t, ctx = _inputs(2, 2, 40, 9, 10, 64)
    dy = torch.randn(2, 40, 10, device=DEV)
    full = _run(m, x, t, ctx, dy)
    for n, p in m.named_parameters():
        if n.startswith("blocks.") == (frozen == "blocks") and not n.startswith("final_layer"):
            p.requires_grad_(False)
    calls = []
    for fn in ("_wgrad", "_dgrad", "_bgrad", "_linear_small_bwd"):
        orig = getattr(dit_grad, fn)
        monkeypatch.setattr(dit_grad, fn, lambda *a, _f=orig, _n=fn, **k: (calls.append(_n), _f(*a, **k))[1])
    for p in m.parameters():
        p.grad = None
    dit_grad.model_forward(m, x, t, ctx).backward(dy)
    if frozen == "blocks":                # the stem's fc2 and xyz projection: one wgrad each and one shared bias sum
        assert calls.count("_wgrad") == 2 and calls.count("_bgrad") == 1, calls
        for n in ("x_embedder.fc2.weight", "xyz_pos_embed.xyz_projection.weight", "t_embedder.mlp.0.weight",
                  "x_embedder.fc1.weight", "pooled_vec_embedder.0.weight", "x_embedder.fc2.bias",
                  "xyz_pos_embed.xyz_projection.bias"):
            assert torch.equal(dict(m.named_parameters())[n].grad, full[n]), n
    else:                                 # no stem backward; each block's seven weight GEMMs
        assert calls.count("_linear_small_bwd") == 0 and calls.count("_wgrad") == 7 * 2, calls
        for n in ("blocks.0.attn.qkv.weight", "blocks.1.mlp.mlp.0.weight", "final_layer.linear.weight"):
            assert torch.equal(dict(m.named_parameters())[n].grad, full[n]), n


@pytest.mark.parametrize("trainable", ["adaLN", "adaLN_and_tokens", "t_embedder", "pooled"])
def test_partly_frozen_stem(trainable):
    """Any subset of the stem's parameters trains: each gets the full run's gradient bits, the frozen ones none."""
    from gaussiananything_b200 import dit_grad
    m = _model(2, True, 128, 2, 64, 10, 2)
    x, t, ctx = _inputs(2, 2, 40, 9, 10, 64)
    dy = torch.randn(2, 40, 10, device=DEV)
    full = _run(m, x, t, ctx, dy)
    keep = {"adaLN": ("adaLN_modulation.",), "adaLN_and_tokens": ("adaLN_modulation.", "x_embedder.", "xyz_pos_embed."),
            "t_embedder": ("t_embedder.",), "pooled": ("pooled_vec_embedder.",)}[trainable]
    stem = {id(p) for p in dit_grad.stem_parameters(m)}
    for n, p in m.named_parameters():
        p.grad = None
        if id(p) in stem and not n.startswith(keep):
            p.requires_grad_(False)
    dit_grad.model_forward(m, x, t, ctx).backward(dy)
    for n, p in m.named_parameters():
        if id(p) not in stem:
            continue
        if n.startswith(keep):
            assert p.grad is not None and torch.equal(p.grad, full[n]), n
        else:
            assert p.grad is None, n


def test_in_place_change_and_double_backward_raise():
    from gaussiananything_b200 import dit_grad
    m = _model(1, False, 128, 2, 64, 3, 1)
    x, t, ctx = _inputs(1, 2, 20, 5, 3, 64)
    y = dit_grad.model_forward(m, x, t, ctx)
    with torch.no_grad():
        m.adaLN_modulation[1].weight.mul_(2)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        y.sum().backward()
    y = dit_grad.model_forward(m, x, t, ctx)
    with torch.no_grad():
        m.final_layer.linear.weight.mul_(2)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        y.sum().backward()
    xs = x.clone().requires_grad_(True)
    y = dit_grad.model_forward(m, xs, t, ctx)
    with pytest.raises(RuntimeError, match="double backward"):
        torch.autograd.grad(y.sum(), xs, create_graph=True)


@pytest.mark.timeout(900)
def test_flow_matching_training_lowers_the_loss():
    """Transport.training_losses on model_forward with AdamW and gradient clipping under bf16 autocast, 20 steps on one
    fixed batch (the same t and noise each step); afterwards the inference engine, rebuilt from the trained weights,
    agrees with model_forward."""
    from gaussiananything_b200 import dit_grad
    from gaussiananything_b200.transport import create_transport
    m = _model(1, False, 128, 2, 64, 3, 2)
    x1, t, ctx = _inputs(1, 4, 64, 16, 3, 64)
    with torch.no_grad():
        y0 = m.eval()(x1, t, ctx)
    eng = m._engine
    m.train()
    transport = create_transport("Linear", "velocity")
    fn = functools.partial(dit_grad.model_forward, m)
    opt = torch.optim.AdamW(m.parameters(), lr=1e-3, weight_decay=0.05)
    losses = []
    for _ in range(20):
        torch.manual_seed(11)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = transport.training_losses(fn, x1, dict(context=ctx))["loss"].mean()
        opt.zero_grad()
        loss.backward()
        torch.nn.utils.clip_grad_norm_(m.parameters(), 1.0)
        opt.step()
        losses.append(float(loss))
    assert all(math.isfinite(v) for v in losses)
    assert losses[-1] < 0.9 * losses[0], losses
    assert m._engine is eng                                  # training never touched the inference engine
    m.eval()
    with torch.no_grad():
        y1 = m(x1, t, ctx)
        want = dit_grad.model_forward(m, x1, t, ctx)
    assert m._engine is not eng                              # the parameters' versions moved: the engine repacked
    assert MR.rel_l2(y1, want) < 6e-3 and MR.rel_l2(y1, y0) > 1e-2
