"""CPU restatement (plain torch, fp32) of the deployed DiT denoiser forward.

TEST INFRASTRUCTURE ONLY (checker for tests/, smoke() and bench.py's CPU leg).
Pinned: tests/test_oracle_dit.py checks this file against golden vectors that
tests/golden/make_dit_golden.py produced by running the reference's own
dit/dit_i23d.py + dit/dit_models_xformers.py code (third-party xformers / timm
ops stubbed by their published semantics).

Follows:
  DiT_I23D_PCD_PixelArt_noclip.forward           /root/reference/dit/dit_i23d.py:511-567
  ..._noclip_clay_stage2.forward                 /root/reference/dit/dit_i23d.py:707-750
  ImageCondDiTBlockPixelArtRMSNormClayLRM.forward /root/reference/dit/dit_models_xformers.py:765-787
  MemEffAttention / Attention                    /root/reference/vit/vision_transformer.py:177-303
  MemoryEfficientCrossAttention                  /root/reference/ldm/modules/attention.py:484-561
  RMSNorm                                        /root/reference/dit/norm.py:27-40
  TimestepEmbedder, T2IFinalLayer                /root/reference/dit/dit_models_xformers.py:62-128
  XYZPosEmbed / Embedder                         /root/reference/vit/vit_triplane.py:187-229, utils/nerf_utils.py:17-65
  forward_with_cfg                               /root/reference/dit/dit_i23d.py:159-172
`sd` is a state_dict in the reference's key layout (SURVEY.md App. B).
"""
import math

import torch
import torch.nn.functional as F


def rmsnorm(x, w, eps=1e-5):
    var = x.float().pow(2).mean(-1, keepdim=True)
    return x * torch.rsqrt(var + eps) * w


def timestep_embedding(t, dim=256, max_period=10000):
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(half, dtype=torch.float32) / half)
    args = t[:, None].float() * freqs[None]
    return torch.cat([torch.cos(args), torch.sin(args)], dim=-1)


def xyz_posenc(xyz, multires=10):
    out = [xyz]
    for k in range(multires):
        f = 2.0 ** k
        out += [torch.sin(xyz * f), torch.cos(xyz * f)]
    return torch.cat(out, -1)


def _heads(x, H):
    B, L, C = x.shape
    return x.view(B, L, H, C // H).transpose(1, 2)          # B H L d


_EMU = False          # when True, round every tensor-core operand to bf16 like the CUDA path does


def _r(x):
    return x.to(torch.bfloat16).to(torch.float32) if _EMU else x


def attention(q, k, v):
    if not _EMU:
        return F.scaled_dot_product_attention(q, k, v)        # softmax(q k^T / sqrt(d)) v
    q, k, v = _r(q), _r(k), _r(v)
    s = (q @ k.transpose(-1, -2)) / math.sqrt(q.shape[-1])
    p = torch.exp(s - s.max(-1, keepdim=True).values)
    return _r((_r(p) @ v) / p.sum(-1, keepdim=True))          # unnormalised P is the bf16 MMA operand


def block_forward(sd, p, x, t0, ctx, H):
    B, N, D = x.shape
    mod = sd[p + "scale_shift_table"][None] + t0.reshape(B, 6, -1)
    s_msa, c_msa, g_msa, s_mlp, c_mlp, g_mlp = mod.chunk(6, dim=1)
    # cross attention on the image tokens (pre-norm + residual)
    h = _r(rmsnorm(x, sd[p + "prenorm_ca_dino.weight"]))
    ctx = _r(ctx)
    q = F.linear(h, sd[p + "cross_attn_dino.to_q.weight"])
    k = F.linear(ctx, sd[p + "cross_attn_dino.to_k.weight"])
    v = F.linear(ctx, sd[p + "cross_attn_dino.to_v.weight"])
    q, k, v = _heads(q, H), _heads(k, H), _heads(v, H)
    q = rmsnorm(q, sd[p + "cross_attn_dino.q_norm.weight"])
    k = rmsnorm(k, sd[p + "cross_attn_dino.k_norm.weight"])
    o = attention(q, k, v).transpose(1, 2).reshape(B, N, D)
    x = x + F.linear(o, sd[p + "cross_attn_dino.to_out.0.weight"], sd[p + "cross_attn_dino.to_out.0.bias"])
    # gated self attention
    h = _r(rmsnorm(x, sd[p + "norm1.weight"]) * (1 + c_msa) + s_msa)
    qkv = F.linear(h, sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"])
    qkv = qkv.view(B, N, 3, H, D // H).permute(2, 0, 3, 1, 4)  # "(K H D)": K outermost
    q, k, v = qkv[0], qkv[1], qkv[2]
    q = rmsnorm(q, sd[p + "attn.q_norm.weight"])
    k = rmsnorm(k, sd[p + "attn.k_norm.weight"])
    o = attention(q, k, v).transpose(1, 2).reshape(B, N, D)
    x = x + g_msa * F.linear(o, sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"])
    # gated FFN (xformers FusedMLP: exact GELU)
    h = _r(rmsnorm(x, sd[p + "norm2.weight"]) * (1 + c_mlp) + s_mlp)
    h = _r(F.gelu(F.linear(h, sd[p + "mlp.mlp.0.weight"]) + sd[p + "mlp.mlp.1.bias"]))
    h = F.linear(h, sd[p + "mlp.mlp.2.weight"]) + sd[p + "mlp.mlp.3.bias"]
    return x + g_mlp * h


def forward(sd, x, t, context, num_heads, depth, return_acts=False, emulate_bf16=False):
    """x [B,N,Cin] fp32, t [B], context dict(img_crossattn [B,M,Dc], img_vector [B,Dc], optional fps-xyz [B,N,3]).
    emulate_bf16: round the tensor-core operands (activations feeding GEMMs / attention) to bf16, which is what
    the reference's bf16 autocast and the CUDA path both do; weights are expected to be bf16-representable."""
    global _EMU
    _EMU = bool(emulate_bf16)
    try:
        return _forward(sd, x, t, context, num_heads, depth, return_acts)
    finally:
        _EMU = False


def _forward(sd, x, t, context, num_heads, depth, return_acts):
    sd = {k: v.float() for k, v in sd.items()}
    ctx = context["img_crossattn"].float()
    vec = context["img_vector"].float()
    temb = F.linear(timestep_embedding(t), sd["t_embedder.mlp.0.weight"], sd["t_embedder.mlp.0.bias"])
    temb = F.linear(F.silu(temb), sd["t_embedder.mlp.2.weight"], sd["t_embedder.mlp.2.bias"])
    pooled = F.layer_norm(vec, vec.shape[-1:], sd["pooled_vec_embedder.0.weight"], sd["pooled_vec_embedder.0.bias"], 1e-5)
    pooled = F.linear(pooled, sd["pooled_vec_embedder.1.weight"], sd["pooled_vec_embedder.1.bias"])
    tt = temb + pooled
    t0 = F.linear(F.silu(tt), sd["adaLN_modulation.1.weight"], sd["adaLN_modulation.1.bias"])
    stage2 = "fps-xyz" in context and (sd["x_embedder.fc1.weight"].shape[1] != x.shape[-1]
                                       or "xyz_pos_embed.xyz_projection.weight" in sd)
    xin = x.float()
    use_pe = "xyz_pos_embed.xyz_projection.weight" in sd
    if stage2 and not use_pe:
        xin = torch.cat([context["fps-xyz"].float(), xin], dim=-1)
    h = _r(F.gelu(F.linear(xin, sd["x_embedder.fc1.weight"], sd["x_embedder.fc1.bias"]), approximate="tanh"))
    h = F.linear(h, sd["x_embedder.fc2.weight"], sd["x_embedder.fc2.bias"])
    if stage2 and use_pe:
        h = h + F.linear(_r(xyz_posenc(context["fps-xyz"].float())), sd["xyz_pos_embed.xyz_projection.weight"],
                         sd["xyz_pos_embed.xyz_projection.bias"])
    acts = {}
    for i in range(depth):
        h = block_forward(sd, "blocks.%d." % i, h, t0, ctx, num_heads)
        acts["block%d" % i] = h
    shift, scale = (sd["final_layer.scale_shift_table"][None] + tt[:, None]).chunk(2, dim=1)
    y = F.layer_norm(h, h.shape[-1:], None, None, 1e-6) * (1 + scale) + shift
    y = F.linear(y, sd["final_layer.linear.weight"], sd["final_layer.linear.bias"]).float().contiguous()
    return (y, acts) if return_acts else y


def forward_with_cfg(sd, x, t, context, cfg_scale, num_heads, depth, emulate_bf16=False):
    eps = forward(sd, x, t, context, num_heads, depth, emulate_bf16=emulate_bf16)
    cond, uncond = torch.split(eps, len(eps) // 2, dim=0)
    half = uncond + cfg_scale * (cond - uncond)
    return torch.cat([half, half], dim=0)


def load_golden(path):
    """Reads a tests/golden/dit_*.npz written by make_dit_golden.py."""
    from oracle.golden_io import load_parts
    z = load_parts(path)
    sd = {k[4:]: torch.from_numpy(z[k].copy()).view(torch.bfloat16).float() for k in z if k.startswith("sd__")}
    ctx = {k[5:]: torch.from_numpy(z[k]) for k in z if k.startswith("ctx__")}
    acts = {k[5:]: torch.from_numpy(z[k]) for k in z if k.startswith("act__")}
    meta = [int(v) for v in z["meta"]]
    cfg = dict(depth=meta[0], hidden=meta[1], heads=meta[2], cin=meta[3], ctx_dim=meta[4], stage2=bool(meta[5]),
               use_pe=bool(meta[6]))
    return dict(sd=sd, ctx=ctx, acts=acts, cfg=cfg, x=torch.from_numpy(z["x"]), t=torch.from_numpy(z["t"]),
                y=torch.from_numpy(z["y"]), y_cfg=torch.from_numpy(z["y_cfg"]),
                traj_euler=torch.from_numpy(z["traj_euler"]), traj_heun=torch.from_numpy(z["traj_heun"]))
