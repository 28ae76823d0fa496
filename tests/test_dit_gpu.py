"""GPU parity tests of the DiT path: wgmma GEMM epilogues, wgmma attention, row kernels (each against a
plain torch fp32 reference of the same op on bf16-rounded inputs), then the whole denoiser and the sampler
against the oracle on the golden vectors generated from the reference's own code.

Tolerances: operands are bf16 (as under the reference's autocast), accumulation fp32.  Against the
bf16-emulating oracle (same operands rounded) the bar is 6e-3 rel-L2 (1.5 bf16 eps); against the fp32 golden 2e-2.
BASELINE.json's 1e-4 is only reachable with fp32 operands."""
import ctypes as C
import math
import os

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(180)]
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def _env():
    from gaussiananything_b200 import dit
    L = dit._bind()
    dev = torch.device("cuda:0")
    st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    return dit, L, dev, st


def _gemm(dit, L, st, A, W, epi, bn):
    M, K = A.shape
    N = W.shape[0]
    rc = L.ga_gemm_bf16_tn(dit._p(A), K, dit._p(W), K, M, N, K, C.byref(epi), bn, st)
    assert rc == 0, rc
    torch.cuda.synchronize()


@pytest.mark.parametrize("M,N,K,bn", [(128, 128, 64, 128), (128, 64, 16, 64), (256, 256, 256, 128),
                                      (1000, 768, 768, 128), (4096, 3072, 768, 256), (200, 192, 1024, 64),
                                      (4096, 768, 3072, 192), (300, 500, 136, 192)])
def test_gemm_bias_bf16(M, N, K, bn):
    dit, L, dev, st = _env()
    torch.manual_seed(M + N + K)
    A = torch.randn(M, K, device=dev).bfloat16()
    W = (torch.randn(N, K, device=dev) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device=dev)
    out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
    e = dit.GaGemmEpilogue(mode=dit.EPI_BF16, bias=bias.data_ptr(), out=out.data_ptr(), ld_out=N)
    _gemm(dit, L, st, A, W, e, bn)
    ref = A.float() @ W.float().T + bias
    assert rel(out.float(), ref) < 4e-3, rel(out.float(), ref)


def test_gemm_epilogues():
    dit, L, dev, st = _env()
    torch.manual_seed(0)
    B, Ntok, D, H = 2, 200, 256, 4
    M, K = B * Ntok, D
    A = torch.randn(M, K, device=dev).bfloat16()
    W = (torch.randn(4 * D, K, device=dev) / math.sqrt(K)).bfloat16()
    bias = torch.randn(4 * D, device=dev) * 0.1
    ref = A.float() @ W.float().T + bias
    # GELU
    out = torch.zeros(M, 4 * D, device=dev, dtype=torch.bfloat16)
    _gemm(dit, L, st, A, W, dit.GaGemmEpilogue(mode=dit.EPI_GELU_BF16, bias=bias.data_ptr(), out=out.data_ptr(), ld_out=4 * D), 128)
    assert rel(out.float(), torch.nn.functional.gelu(ref)) < 4e-3
    # fp32 out
    o32 = torch.zeros(M, 4 * D, device=dev)
    _gemm(dit, L, st, A, W, dit.GaGemmEpilogue(mode=dit.EPI_F32, bias=bias.data_ptr(), out=o32.data_ptr(), ld_out=4 * D), 128)
    assert rel(o32, ref) < 1e-5
    # gated residual, in place, gate per batch item
    Wd = W[:D].contiguous()
    x0 = torch.randn(M, D, device=dev)
    x = x0.clone()
    mod = torch.randn(B, 6 * D, device=dev)
    gate = mod[:, 2 * D:3 * D]
    _gemm(dit, L, st, A, Wd, dit.GaGemmEpilogue(mode=dit.EPI_RESID_GATE_F32, bias=bias.data_ptr(), out=x.data_ptr(), ld_out=D,
                                                 gate=gate.data_ptr(), gate_ld=6 * D, rows_per_batch=Ntok), 128)
    want = x0 + gate.repeat_interleave(Ntok, 0) * ref[:, :D]
    assert rel(x, want) < 1e-5
    # the same with 128 x 192 tiles (the width the engine picks for the N = 768 residual GEMMs); 192 has no HEADS mode
    x = x0.clone()
    _gemm(dit, L, st, A, Wd, dit.GaGemmEpilogue(mode=dit.EPI_RESID_GATE_F32, bias=bias.data_ptr(), out=x.data_ptr(), ld_out=D,
                                                 gate=gate.data_ptr(), gate_ld=6 * D, rows_per_batch=Ntok), 192)
    assert rel(x, want) < 1e-5
    bad = dit.GaGemmEpilogue(mode=dit.EPI_HEADS, heads=H)
    assert L.ga_gemm_bf16_tn(dit._p(A), K, dit._p(W), K, M, 3 * D, K, C.byref(bad), 192, st) != 0
    # heads: q,k normed + v transposed
    Np = 256
    W3 = W[:3 * D].contiguous()
    q = torch.zeros(B * H, Np, 64, device=dev, dtype=torch.bfloat16)
    k = torch.zeros_like(q)
    vt = torch.zeros(B * H, 64, Np, device=dev, dtype=torch.bfloat16)
    qn, kn = torch.rand(64, device=dev) + 0.5, torch.rand(64, device=dev) + 0.5
    e = dit.GaGemmEpilogue(mode=dit.EPI_HEADS, bias=bias.data_ptr(), q=q.data_ptr(), k=k.data_ptr(), vt=vt.data_ptr(),
                           qn_w=qn.data_ptr(), kn_w=kn.data_ptr(), heads=H, first_part=0, tok_pitch=Np,
                           rows_per_batch=Ntok, eps=1e-5)
    _gemm(dit, L, st, A, W3, e, 128)
    r3 = ref[:, :3 * D].view(B, Ntok, 3, H, 64).permute(2, 0, 3, 1, 4)          # K B H L D
    rms = lambda t, w: t * torch.rsqrt(t.pow(2).mean(-1, keepdim=True) + 1e-5) * w
    assert rel(q.view(B, H, Np, 64)[:, :, :Ntok].float(), rms(r3[0], qn)) < 4e-3
    assert rel(k.view(B, H, Np, 64)[:, :, :Ntok].float(), rms(r3[1], kn)) < 4e-3
    assert rel(vt.view(B, H, 64, Np)[:, :, :, :Ntok].float(), r3[2].transpose(-1, -2)) < 4e-3
    assert float(q.view(B, H, Np, 64)[:, :, Ntok:].abs().max()) == 0.0          # padding untouched


@pytest.mark.parametrize("static_bound", [False, True])
@pytest.mark.parametrize("B,H,Nq,Nk", [(1, 1, 128, 128), (2, 3, 200, 1369), (1, 2, 768, 768), (2, 12, 2048, 2048)])
def test_attention(B, H, Nq, Nk, static_bound):
    dit, L, dev, st = _env()
    torch.manual_seed(Nq + Nk)
    pq, pk = (Nq + 127) // 128 * 128, (Nk + 127) // 128 * 128
    q = torch.zeros(B * H, pq, 64, device=dev, dtype=torch.bfloat16)
    k = torch.zeros(B * H, pk, 64, device=dev, dtype=torch.bfloat16)
    vt = torch.zeros(B * H, 64, pk, device=dev, dtype=torch.bfloat16)
    q[:, :Nq] = torch.randn(B * H, Nq, 64, device=dev) * 1.2
    k[:, :Nk] = torch.randn(B * H, Nk, 64, device=dev) * 1.2
    vt[:, :, :Nk] = torch.randn(B * H, 64, Nk, device=dev)
    out = torch.zeros(B, Nq, H * 64, device=dev, dtype=torch.bfloat16)
    # static mode: a valid upper bound of |q.k|/8 (here Cauchy-Schwarz on the actual norms); 0 = online softmax
    bound = float(q.float().norm(dim=-1).max() * k.float().norm(dim=-1).max()) / 8.0 if static_bound else 0.0
    if static_bound:
        assert bound <= 40.0
    rc = L.ga_attention_bf16(dit._p(q), dit._p(k), dit._p(vt), dit._p(out), B, H, Nq, Nk, pq, pk, 0.125, bound, st)
    assert rc == 0, rc
    torch.cuda.synchronize()
    ref = torch.nn.functional.scaled_dot_product_attention(
        q[:, :Nq].float().view(B, H, Nq, 64), k[:, :Nk].float().view(B, H, Nk, 64),
        vt[:, :, :Nk].float().transpose(-1, -2).reshape(B, H, Nk, 64))
    ref = ref.transpose(1, 2).reshape(B, Nq, H * 64)
    assert rel(out.float(), ref) < 6e-3, rel(out.float(), ref)


def test_attention_bound_too_large_falls_back_to_online_softmax():
    """score_bound > 40 (or <= 0) must take the running-maximum path: large logits stay exact."""
    dit, L, dev, st = _env()
    torch.manual_seed(5)
    B, H, N = 1, 2, 256
    q = (torch.randn(B * H, N, 64, device=dev) * 4.0).bfloat16()
    k = (torch.randn(B * H, N, 64, device=dev) * 4.0).bfloat16()
    vt = torch.randn(B * H, 64, N, device=dev).bfloat16()
    ref = torch.nn.functional.scaled_dot_product_attention(
        q.float().view(B, H, N, 64), k.float().view(B, H, N, 64), vt.float().transpose(-1, -2).reshape(B, H, N, 64))
    ref = ref.transpose(1, 2).reshape(B, N, H * 64)
    for bound in (0.0, 500.0):
        out = torch.zeros(B, N, H * 64, device=dev, dtype=torch.bfloat16)
        assert L.ga_attention_bf16(dit._p(q), dit._p(k), dit._p(vt), dit._p(out), B, H, N, N, N, N, 0.125, bound, st) == 0
        torch.cuda.synchronize()
        assert rel(out.float(), ref) < 8e-3, (bound, rel(out.float(), ref))


def test_row_kernels():
    dit, L, dev, st = _env()
    torch.manual_seed(1)
    B, Ntok, D = 2, 77, 256
    R = B * Ntok
    x = torch.randn(R, D, device=dev)
    w = torch.rand(D, device=dev) + 0.5
    mod = torch.randn(B, 6 * D, device=dev)
    out = torch.zeros(R, D, device=dev, dtype=torch.bfloat16)
    assert L.ga_rmsnorm_modulate(dit._p(x), dit._p(w), dit._p(mod[:, :D]), dit._p(mod[:, D:2 * D]), 6 * D, Ntok, dit._p(out), R, D, 1e-5, st) == 0
    ref = x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-5) * w
    ref = ref * (1 + mod[:, D:2 * D].repeat_interleave(Ntok, 0)) + mod[:, :D].repeat_interleave(Ntok, 0)
    torch.cuda.synchronize()
    assert rel(out.float(), ref) < 3e-3
    # small linear with SiLU in/out + accumulate
    xin = torch.randn(B, 300, device=dev); W = torch.randn(40, 300, device=dev) / 17; b = torch.randn(40, device=dev)
    y = torch.ones(B, 40, device=dev)
    assert L.ga_linear_small(dit._p(xin), dit._p(W), dit._p(b), dit._p(y), B, 40, 300, 1, 1, 1, st) == 0
    torch.cuda.synchronize()
    want = 1 + torch.nn.functional.silu(torch.nn.functional.silu(xin) @ W.T + b)
    assert rel(y, want) < 1e-5
    # final layer
    Cout = 10
    modf = torch.randn(B, 2 * D, device=dev) * 0.3
    Wf = torch.randn(Cout, D, device=dev) / 16; bf = torch.randn(Cout, device=dev)
    yo = torch.zeros(R, Cout, device=dev)
    assert L.ga_final_layer(dit._p(x), dit._p(modf), dit._p(Wf), dit._p(bf), dit._p(yo), R, D, Cout, Ntok, 1e-6, st) == 0
    torch.cuda.synchronize()
    ln = torch.nn.functional.layer_norm(x, (D,), None, None, 1e-6)
    h = ln * (1 + modf[:, D:].repeat_interleave(Ntok, 0)) + modf[:, :D].repeat_interleave(Ntok, 0)
    assert rel(yo, h @ Wf.T + bf) < 1e-5


def _build(g, dev):
    from gaussiananything_b200 import dit
    c = g["cfg"]
    cls = dit.DiT_I23D_PCD_PixelArt_noclip_clay_stage2 if c["stage2"] else dit.DiT_I23D_PCD_PixelArt_noclip
    kw = dict(use_pe_cond=c["use_pe"]) if c["stage2"] else {}
    m = cls(input_size=32, num_classes=0, learn_sigma=False, in_channels=c["cin"], context_dim=c["ctx_dim"],
            roll_out=True, pooling_ctx_dim=768, patch_size=1, depth=c["depth"], hidden_size=c["hidden"],
            num_heads=c["heads"], use_clay_ca=True, **kw)
    missing, unexpected = m.load_state_dict(g["sd"], strict=False)
    assert not unexpected
    assert all(any(u in k for u in ("clip_spatial_proj", "cap_embedder", "attention_y_norm")) for k in missing), missing
    return m.to(dev).eval()


@pytest.mark.parametrize("name", ["dit_stage1_small", "dit_stage2_small", "dit_stage2_concat_small"])
def test_dit_forward_matches_oracle_and_reference_golden(name):
    from oracle import dit_oracle as do
    g = do.load_golden(os.path.join(GOLD, name + ".npz"))
    c = g["cfg"]
    dev = torch.device("cuda:0")
    m = _build(g, dev)
    ctx = {k: v.to(dev) for k, v in g["ctx"].items()}
    y = m(g["x"].to(dev), g["t"].to(dev), ctx)
    assert y.dtype == torch.float32 and y.shape == g["y"].shape
    ye = do.forward(g["sd"], g["x"], g["t"], g["ctx"], c["heads"], c["depth"], emulate_bf16=True)
    # 1.5 x bf16 epsilon: the oracle rounds the same operands but not at bit-identical points (e.g. the kernel's
    # unnormalised P uses a static bound instead of the row maximum)
    assert rel(y.cpu(), ye) < 6e-3, ("vs bf16-emulating oracle", rel(y.cpu(), ye))
    assert rel(y.cpu(), g["y"]) < 2e-2, ("vs reference fp32 golden", rel(y.cpu(), g["y"]))
    yc = m.forward_with_cfg(g["x"].to(dev), g["t"].to(dev), ctx, 4.0)
    assert rel(yc.cpu(), g["y_cfg"]) < 3e-2
    half = yc.shape[0] // 2
    assert torch.equal(yc[:half], yc[half:])
    # graph replay == eager launches
    m._engine.use_graph = False
    y2 = m(g["x"].to(dev), g["t"].to(dev), ctx)
    assert torch.equal(y, y2)


def test_sampler_on_gpu_matches_reference_trajectory():
    from oracle import dit_oracle as do
    from gaussiananything_b200 import transport as tr
    g = do.load_golden(os.path.join(GOLD, "dit_stage1_small.npz"))
    dev = torch.device("cuda:0")
    m = _build(g, dev)
    ctx = {k: v.to(dev) for k, v in g["ctx"].items()}
    s = tr.Sampler(tr.create_transport("GVP", "velocity", None, None, None, "lognorm"))
    traj = s.sample_ode(sampling_method="euler", num_steps=5)(g["x"].to(dev), m.forward_with_cfg, context=ctx, cfg_scale=4.0)
    assert traj.shape == g["traj_euler"].shape
    assert rel(traj.cpu(), g["traj_euler"]) < 2e-2


def test_dit_b_full_size_properties():
    """DiT-PixArt-PCD-CLAY-B at BASELINE config C3 size (N=2048): finite, deterministic, CFG identity at s=1."""
    from gaussiananything_b200 import dit
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    m = dit.DiT_models["DiT-PixArt-PCD-CLAY-B"](input_size=32, num_classes=0, learn_sigma=False, in_channels=3,
                                                context_dim=1024, roll_out=True, pooling_ctx_dim=768)
    m.randomize_zero_init_().to(dev).eval()
    B, N, M = 2, 2048, 1369
    x = torch.randn(B, N, 3, device=dev)
    t = torch.rand(B, device=dev)
    ctx = {"img_crossattn": torch.randn(B, M, 1024, device=dev), "img_vector": torch.randn(B, 1024, device=dev)}
    y1 = m(x, t, ctx)
    y2 = m(x, t, ctx)
    assert torch.isfinite(y1).all() and torch.equal(y1, y2) and float(y1.abs().mean()) > 0
    yc = m.forward_with_cfg(x, t, ctx, 1.0)              # s = 1 -> exactly the conditional half
    assert rel(yc[0], y1[0]) < 1e-6
    # batch rows are independent: swapping the two samples swaps the outputs
    ctx_sw = {k: v.flip(0).contiguous() for k, v in ctx.items()}
    y3 = m(x.flip(0).contiguous(), t.flip(0).contiguous(), ctx_sw)
    assert rel(y3.flip(0), y1) < 1e-5


def test_dit_l_c4_size_properties():
    """BASELINE configs[3] size: DiT-L stage 1 and stage 2 at N=4096, d=1024.  The oracle cannot run this in seconds,
    so size-independent properties only: finite, run-to-run identical bits, batch items independent."""
    from gaussiananything_b200 import dit
    dev = torch.device("cuda:0")
    torch.manual_seed(1)
    B, N, M = 2, 4096, 1369
    for name, cin, stage2 in (("DiT-PixArt-PCD-CLAY-L", 3, False), ("DiT-PixArt-PCD-CLAY-stage2-L", 10, True)):
        m = dit.DiT_models[name](input_size=32, num_classes=0, learn_sigma=False, in_channels=cin, context_dim=1024,
                                 roll_out=True, pooling_ctx_dim=768)
        m.randomize_zero_init_().to(dev).eval()
        x = torch.randn(B, N, cin, device=dev)
        t = torch.rand(B, device=dev)
        ctx = {"img_crossattn": torch.randn(B, M, 1024, device=dev), "img_vector": torch.randn(B, 1024, device=dev)}
        if stage2:
            ctx["fps-xyz"] = torch.rand(B, N, 3, device=dev) - 0.5
        y1 = m(x, t, ctx)
        y2 = m(x, t, ctx)
        assert y1.shape == (B, N, cin)
        assert torch.isfinite(y1).all() and torch.equal(y1, y2) and float(y1.abs().mean()) > 0
        ctx_sw = {k: v.flip(0).contiguous() for k, v in ctx.items()}
        y3 = m(x.flip(0).contiguous(), t.flip(0).contiguous(), ctx_sw)
        assert rel(y3.flip(0), y1) < 1e-5
        del m
        torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------
# round 2: context K/V cache safety, per-block activations, C3-size parity, CFG de-duplication, inference-only guard
# ---------------------------------------------------------------------------------------------------------------
def _rand_ctx(B, M, Dc, dev, seed):
    g = torch.Generator().manual_seed(seed)
    return {"img_crossattn": torch.randn(B, M, Dc, generator=g).to(dev), "img_vector": torch.randn(B, Dc, generator=g).to(dev)}


def test_context_kv_cache_is_not_stale_across_samples():
    """Round-1 bug (VERDICT weak #1 / ADVICE high): the cross-attention K/V cache was keyed on data_ptr(); a new
    context allocated at the recycled address of a freed one silently reused the old K/V.  Two DIFFERENT contexts
    of the same shape, the first freed before the second is allocated, must both match the oracle."""
    from oracle import dit_oracle as do
    g = do.load_golden(os.path.join(GOLD, "dit_stage1_small.npz"))
    c = g["cfg"]
    dev = torch.device("cuda:0")
    m = _build(g, dev)
    x, t = g["x"].to(dev), g["t"].to(dev)
    B, M, Dc = g["ctx"]["img_crossattn"].shape
    outs, ptrs = [], []
    for seed in (11, 12, 13):
        ctx = _rand_ctx(B, M, Dc, dev, seed)
        ptrs.append(ctx["img_crossattn"].data_ptr())
        y = m(x, t, ctx).cpu()
        want = do.forward(g["sd"], g["x"], g["t"], {k: v.cpu() for k, v in ctx.items()}, c["heads"], c["depth"],
                          emulate_bf16=True)
        assert rel(y, want) < 6e-3, (seed, rel(y, want))
        outs.append(y)
        del ctx, y                                   # frees the block: the next context usually lands on the same address
    assert not torch.equal(outs[0], outs[1]) and not torch.equal(outs[1], outs[2])
    # same tensor object again: cache hit, same bits; modified in place: version counter invalidates the cache
    ctx = _rand_ctx(B, M, Dc, dev, 21)
    y1 = m(x, t, ctx)
    y2 = m(x, t, ctx)
    assert torch.equal(y1, y2)
    ctx["img_crossattn"].mul_(0.5)
    y3 = m(x, t, ctx)
    want = do.forward(g["sd"], g["x"], g["t"], {k: v.cpu() for k, v in ctx.items()}, c["heads"], c["depth"], emulate_bf16=True)
    assert rel(y3.cpu(), want) < 6e-3 and not torch.equal(y1, y3)


def test_runs_under_inference_mode_like_the_reference_eval_path():
    """The reference samples under @th.inference_mode() (flow_matching_trainer.py:747): inference tensors have no
    version counter, and workspaces allocated inside must stay usable outside."""
    from oracle import dit_oracle as do
    g = do.load_golden(os.path.join(GOLD, "dit_stage1_small.npz"))
    c = g["cfg"]
    dev = torch.device("cuda:0")
    m = _build(g, dev)
    want = None
    with torch.inference_mode():
        x, t = g["x"].to(dev), g["t"].to(dev)
        for seed in (31, 32):
            ctx = _rand_ctx(*g["ctx"]["img_crossattn"].shape, dev, seed)
            y = m.forward_with_cfg(x, t, ctx, 4.0)
            want = do.forward_with_cfg(g["sd"], g["x"], g["t"], {k: v.cpu() for k, v in ctx.items()}, 4.0, c["heads"],
                                       c["depth"], emulate_bf16=True)
            assert rel(y.cpu(), want) < 8e-3
            del ctx
    ctx = {k: v.to(dev) for k, v in g["ctx"].items()}            # engine built under inference mode, used outside it
    y = m(g["x"].to(dev), g["t"].to(dev), ctx)
    assert rel(y.cpu(), g["y"]) < 2e-2


@pytest.mark.parametrize("name", ["dit_stage1_small", "dit_stage2_small"])
def test_per_block_activations_match_reference_golden(name):
    """Residual stream after every block (north_star: parity on DiT activations) against the hooks the golden
    generator put on the reference's own blocks, and against the bf16-emulating oracle."""
    from oracle import dit_oracle as do
    g = do.load_golden(os.path.join(GOLD, name + ".npz"))
    c = g["cfg"]
    dev = torch.device("cuda:0")
    m = _build(g, dev)
    ctx = {k: v.to(dev) for k, v in g["ctx"].items()}
    y0 = m(g["x"].to(dev), g["t"].to(dev), ctx)
    m._engine.tap_blocks = True
    y = m(g["x"].to(dev), g["t"].to(dev), ctx)
    assert torch.equal(y, y0)                                     # tapping does not change the result
    taps = m._engine.s["taps"].cpu()
    _, acts_e = do.forward(g["sd"], g["x"], g["t"], g["ctx"], c["heads"], c["depth"], return_acts=True, emulate_bf16=True)
    B, N = g["x"].shape[:2]
    worst_e = worst_g = 0.0
    for i in range(c["depth"]):
        got = taps[i].reshape(B, N, -1)
        worst_e = max(worst_e, rel(got, acts_e["block%d" % i]))
        worst_g = max(worst_g, rel(got, g["acts"]["block%d" % i]))
    print("per-block rel-L2: vs bf16-emulating oracle %.2e, vs reference fp32 golden %.2e" % (worst_e, worst_g))
    assert worst_e < 4e-3, worst_e
    assert worst_g < 1.5e-2, worst_g


@pytest.mark.timeout(900)
def test_c3_size_forward_and_blocks_vs_oracle():
    """BASELINE configs[2]: DiT-PixArt-PCD-CLAY-B (L12, D768, H12) at N=2048, M=1369, CFG batch 2 -- the whole
    forward and every block's residual stream against the oracle (bf16 operands emulated) at the real size
    (multi-tile GEMMs, 16 key blocks per attention item, ragged 1369-token context)."""
    from gaussiananything_b200 import dit
    from oracle import dit_oracle as do
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    torch.set_num_threads(os.cpu_count() or 1)
    m = dit.DiT_models["DiT-PixArt-PCD-CLAY-B"](input_size=32, num_classes=0, learn_sigma=False, in_channels=3,
                                                context_dim=1024, roll_out=True, pooling_ctx_dim=768)
    m.randomize_zero_init_()
    for p in m.parameters():                                      # bf16-representable weights: the oracle sees the
        p.data.copy_(p.data.to(torch.bfloat16).float())          # exact values the tensor cores multiply
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    m.to(dev).eval()
    B, N, M = 2, 2048, 1369
    x, t = torch.randn(B, N, 3), torch.rand(B)
    ctx = {"img_crossattn": torch.randn(B, M, 1024), "img_vector": torch.randn(B, 1024)}
    dctx = {k: v.to(dev) for k, v in ctx.items()}
    m._engine_for(x.to(dev), dctx).tap_blocks = True
    y = m(x.to(dev), t.to(dev), dctx).cpu()
    taps = m._engine.s["taps"].cpu()
    want, acts = do.forward(sd, x, t, ctx, 12, 12, return_acts=True, emulate_bf16=True)
    worst = max(rel(taps[i].reshape(B, N, -1), acts["block%d" % i]) for i in range(12))
    print("C3 size: output rel-L2 %.2e, worst block %.2e" % (rel(y, want), worst))
    assert rel(y, want) < 6e-3, rel(y, want)
    assert worst < 4e-3, worst
    yc = m.forward_with_cfg(x.to(dev), t.to(dev), dctx, 4.0).cpu()
    c, u = want[:1], want[1:]
    assert rel(yc[:1], u + 4.0 * (c - u)) < 2e-2


def test_cfg_dedup_fast_path_is_bit_identical():
    """SURVEY F13: in the reference's stage-2 call uc == c, so u + s (c - u) == c.  With cfg_dedup=True only B
    rows are evaluated; the result must equal the 2B call bit for bit, and differing halves must not take the path."""
    from oracle import dit_oracle as do
    g = do.load_golden(os.path.join(GOLD, "dit_stage2_small.npz"))
    dev = torch.device("cuda:0")
    m = _build(g, dev)
    h = g["x"].shape[0] // 2
    x = torch.cat([g["x"][:h], g["x"][:h]], 0).to(dev)
    t = torch.cat([g["t"][:h], g["t"][:h]], 0).to(dev)
    ctx = {k: torch.cat([v[:h], v[:h]], 0).to(dev) for k, v in g["ctx"].items()}
    full = m.forward_with_cfg(x, t, ctx, 4.0)
    m.cfg_dedup = True
    fast = m.forward_with_cfg(x, t, ctx, 4.0)
    assert m._engine._shape[0] == h                              # really ran B rows
    assert torch.equal(full, fast)
    # halves differ (stage-1 style: zeroed unconditional tokens): must fall back to the 2B evaluation
    ctx2 = {k: v.clone() for k, v in ctx.items()}
    ctx2["img_crossattn"][h:] = 0
    y2 = m.forward_with_cfg(x, t, ctx2, 4.0)
    m.cfg_dedup = False
    y2_ref = m.forward_with_cfg(x, t, ctx2, 4.0)
    assert torch.equal(y2, y2_ref) and not torch.equal(y2, full)


def test_inference_only_guard_and_parameter_updates():
    from oracle import dit_oracle as do
    g = do.load_golden(os.path.join(GOLD, "dit_stage1_small.npz"))
    dev = torch.device("cuda:0")
    m = _build(g, dev)
    ctx = {k: v.to(dev) for k, v in g["ctx"].items()}
    x, t = g["x"].to(dev), g["t"].to(dev)
    with pytest.raises(RuntimeError, match="inference-only"):
        m(x.clone().requires_grad_(True), t, ctx)
    m.train()
    with pytest.raises(RuntimeError, match="inference-only"):
        m(x, t, ctx)
    with torch.no_grad():
        y0 = m(x, t, ctx)                                         # fine under no_grad even in train mode
    m.eval()
    # an in-place parameter update (optimizer step / .data.copy_) must not leave a stale bf16 pack / CUDA graph
    with torch.no_grad():
        m.final_layer.linear.weight.mul_(2.0)
        m.final_layer.linear.bias.mul_(2.0)
    y1 = m(x, t, ctx)
    assert rel(y1, 2.0 * y0) < 1e-5


@pytest.mark.timeout(2400)
def test_c4_size_forward_vs_oracle():
    """BASELINE configs[3]: DiT-PixArt-PCD-CLAY-L (L24, D1024, H16) at N=4096, M=1369, CFG batch 2 -- stage 1 against
    the oracle with bf16 operands emulated (minutes of CPU time on the GPU box's host cores; the size-independent
    properties of stage 2 at this size are in test_dit_l_c4_size_properties)."""
    from gaussiananything_b200 import dit
    from oracle import dit_oracle as do
    dev = torch.device("cuda:0")
    torch.manual_seed(4)
    torch.set_num_threads(os.cpu_count() or 1)
    m = dit.DiT_models["DiT-PixArt-PCD-CLAY-L"](input_size=32, num_classes=0, learn_sigma=False, in_channels=3,
                                                context_dim=1024, roll_out=True, pooling_ctx_dim=768)
    m.randomize_zero_init_()
    for p in m.parameters():
        p.data.copy_(p.data.to(torch.bfloat16).float())
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    m.to(dev).eval()
    B, N, M = 2, 4096, 1369
    x, t = torch.randn(B, N, 3), torch.rand(B)
    ctx = {"img_crossattn": torch.randn(B, M, 1024), "img_vector": torch.randn(B, 1024)}
    y = m(x.to(dev), t.to(dev), {k: v.to(dev) for k, v in ctx.items()}).cpu()
    with torch.no_grad():
        want = do.forward(sd, x, t, ctx, 16, 24, emulate_bf16=True)
    print("C4 size: output rel-L2 %.2e" % rel(y, want))
    assert rel(y, want) < 8e-3, rel(y, want)
