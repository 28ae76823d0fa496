"""CPU restatement (plain torch, fp32) of the deployed VAE decode path latent tokens -> surfels (SURVEY.md section 8f row N1).

TEST INFRASTRUCTURE ONLY.  Pinned: tests/test_oracle_vae.py checks this file against golden vectors that
tests/golden/make_vae_golden.py produced by running the reference's own code on CPU (third-party xformers / timm ops
stubbed by their published semantics, tests/golden/_ref_stubs.py).  No CUDA path exists for this row yet;
the oracle and the goldens are the first step of building it.

Follows:
  pcd_structured_latent_space_vae_decoder_cascaded            /root/reference/vit/vit_triplane.py:1594-1676
    vit_decode_backbone / forward_vit_decoder                 /root/reference/vit/vit_triplane.py:1415-1427,1546-1547
    vit_decode_postprocess (base + first up-sampler)          /root/reference/vit/vit_triplane.py:1467-1501
    _get_base_gaussians / _gaussian_pred_activations          /root/reference/vit/vit_triplane.py:1388-1440
    activations (offset/opacity/scale/rot/rgb)                /root/reference/vit/vit_triplane.py:1289-1313
  surfel_prediction (SiLU + Linear -> 13)                     /root/reference/vit/vit_triplane.py:287-345
  GS_Adaptive_Read_Write_CA_adaptive_2dgs.forward             /root/reference/vit/vit_triplane.py:991-1064
  DiT2.forward / DiTBlock2.forward / modulate2                /root/reference/dit/dit_decoder.py:15-42,100-160
  DiTBlock (LayerNorm eps 1e-6 no affine, qk-normed MHA, MLP) /root/reference/dit/dit_models_xformers.py:232-300
  SRT Transformer / PreNorm                                   /root/reference/nsr/srt/layers.py:82-90,146-186
  MemEffAttention (qk-norm)                                   /root/reference/vit/vision_transformer.py:177-303
`sd` is the state_dict of the reference decoder (keys vit_decoder.*, superresolution.*).
"""
import torch
import torch.nn.functional as F

from .dit_oracle import _heads, rmsnorm


def _mha(sd, p, x, H):
    """qkv Linear (K H D column layout) -> per-head RMSNorm of q, k -> softmax(q k^T / sqrt d) v -> proj."""
    B, L, D = x.shape
    qkv = F.linear(x, sd[p + "qkv.weight"], sd[p + "qkv.bias"]).view(B, L, 3, H, D // H).permute(2, 0, 3, 1, 4)
    q = rmsnorm(qkv[0], sd[p + "q_norm.weight"])
    k = rmsnorm(qkv[1], sd[p + "k_norm.weight"])
    o = F.scaled_dot_product_attention(q, k, qkv[2]).transpose(1, 2).reshape(B, L, D)
    return F.linear(o, sd[p + "proj.weight"], sd[p + "proj.bias"])


def _fused_mlp(sd, p, x):
    h = F.gelu(F.linear(x, sd[p + "mlp.0.weight"]) + sd[p + "mlp.1.bias"])          # xformers FusedMLP: exact GELU
    return F.linear(h, sd[p + "mlp.2.weight"]) + sd[p + "mlp.3.bias"]


def dit2_forward(sd, c, num_heads, depth, prefix="vit_decoder."):
    """DiT2 with roll_out=True, in_plane_attention=False: x starts as the learned position embedding, the latent
    tokens c condition every block PER TOKEN through adaLN (dit_decoder.py:100-160)."""
    x = sd[prefix + "pos_embed"].expand(c.shape[0], -1, -1)
    D = x.shape[-1]
    for i in range(depth):
        p = "%sblocks.%d." % (prefix, i)
        mod = F.linear(F.silu(c), sd[p + "adaLN_modulation.1.weight"], sd[p + "adaLN_modulation.1.bias"])
        s_msa, c_msa, g_msa, s_mlp, c_mlp, g_mlp = mod.chunk(6, dim=-1)
        h = F.layer_norm(x, (D,), None, None, 1e-6) * (1 + c_msa) + s_msa
        x = x + g_msa * _mha(sd, p + "attn.", h, num_heads)
        h = F.layer_norm(x, (D,), None, None, 1e-6) * (1 + c_mlp) + s_mlp
        x = x + g_mlp * _fused_mlp(sd, p + "mlp.", h)
    return x


class Activations:
    """vit_triplane.py:1289-1313 with rendering_kwargs['sampler_bbox_max'] = scene_max."""

    def __init__(self, scene_max=0.45):
        self.scene_max = float(scene_max)
        self.scaling_factor = self.scene_max * 0.01 / F.softplus(torch.tensor(0.0))

    def offset(self, x):
        return torch.tanh(x) * self.scene_max * 0.5

    def pack(self, pos, x):
        return torch.cat([pos, torch.sigmoid(x[..., 3:4]), F.softplus(x[..., 4:6]) * self.scaling_factor,
                          F.normalize(x[..., 6:10], dim=-1), 0.5 * torch.tanh(x[..., 10:]) + 0.5], dim=-1)


def srt_transformer(sd, p, x, heads, depth):
    D = x.shape[-1]
    for l in range(depth):
        q = "%slayers.%d." % (p, l)
        h = F.layer_norm(x, (D,), sd[q + "0.norm.weight"], sd[q + "0.norm.bias"], 1e-5)
        x = _mha(sd, q + "0.fn.", h, heads) + x
        h = F.layer_norm(x, (D,), sd[q + "1.norm.weight"], sd[q + "1.norm.bias"], 1e-5)
        x = _fused_mlp(sd, q + "1.fn.", h) + x
    return x


def upsample(sd, p, tokens, base_gaussians, base_pre, act, depth):
    """One cascade stage: every token spawns f children.  tokens [B,N,C], base_gaussians / base_pre [B,N,13].
    Returns (gaussians [B,N*f,13], pre-activations [B,N*f,13], child embeddings [B,N*f,C])."""
    B, N, C = tokens.shape
    emb = sd[p + "latent_embedding"]                                   # [1, f, C]
    f = emb.shape[1]
    seq = torch.cat([tokens.reshape(B * N, 1, C), emb.expand(B * N, -1, -1)], dim=1)
    seq = srt_transformer(sd, p + "transformer.", seq, C // 64, depth)[:, 1:].reshape(B, N, f, C)
    h = F.layer_norm(seq, (C,), sd[p + "gaussian_residual_pred.norm.weight"], sd[p + "gaussian_residual_pred.norm.bias"], 1e-5)
    res = F.linear(h, sd[p + "gaussian_residual_pred.fn.weight"], sd[p + "gaussian_residual_pred.fn.bias"])
    pos = act.offset(res[..., :3]) + base_gaussians[..., None, :3]
    pre = res + base_pre[:, :, None, :]
    g = act.pack(pos, pre).float()
    return g.reshape(B, N * f, 13), pre.reshape(B, N * f, 13), seq.reshape(B, N * f, C)


def decode(sd, latent, query_xyz, num_heads, depth, scene_max=0.45, skip_weight=0.1):
    """latent [B,N,Cz] (the 'latent_normalized' tokens), query_xyz [B,N,3] anchor points.  Returns a dict with every
    stage the reference exposes (vit_decode_backbone + vit_decode_postprocess + forward_gaussians)."""
    sd = {k: v.float() for k, v in sd.items()}
    act = Activations(scene_max)
    q = "superresolution."
    # post_quant_conv: timm Mlp with tanh-GELU (vit_triplane.py:88,1323-1326)
    x0 = F.linear(F.gelu(F.linear(latent, sd[q + "post_quant_conv.fc1.weight"], sd[q + "post_quant_conv.fc1.bias"]),
                         approximate="tanh"), sd[q + "post_quant_conv.fc2.weight"], sd[q + "post_quant_conv.fc2.bias"])
    tok = dit2_forward(sd, x0, num_heads, depth)
    base_pre = F.linear(F.silu(tok), sd[q + "conv_sr.gaussian_pred.1.weight"], sd[q + "conv_sr.gaussian_pred.1.bias"])
    base = act.pack(act.offset(base_pre[..., :3]) * skip_weight + query_xyz, base_pre)
    up1_depth = depth // 6 if depth == 12 else 2                       # vit_triplane.py:1340
    g1, pre1, emb1 = upsample(sd, q + "ada_CA_f4_1.", tok, base, base_pre, act, up1_depth)
    g2, pre2, emb2 = upsample(sd, q + "ada_CA_f4_2.", emb1, g1, pre1, act, 1)
    g3, _, _ = upsample(sd, q + "ada_CA_f4_3.", emb2, g2, pre2, act, 1)
    return {"post_quant": x0, "latent_from_vit": tok, "base_pre_activate": base_pre, "gaussians_base": base,
            "gaussians_upsampled": g1, "gaussians_upsampled_2": g2, "gaussians_upsampled_3": g3,
            "gaussians": g1}                                           # forward_gaussians: "only adopt SR"


def load_golden(path):
    from oracle.golden_io import load_parts
    z = load_parts(path)
    sd = {}
    for k in z:
        if k.startswith("w:"):
            bits = torch.from_numpy(z[k].astype("int32")).to(torch.int32) << 16
            sd[k[2:]] = bits.view(torch.float32)
        elif k.startswith("f:"):
            sd[k[2:]] = torch.from_numpy(z[k])
    D, depth, heads, zc, B, N = [int(v) for v in z["meta"]]
    out = {k[4:]: torch.from_numpy(z[k]) for k in z if k.startswith("out_")}
    return dict(sd=sd, D=D, depth=depth, heads=heads, latent=torch.from_numpy(z["in_latent"]),
                xyz=torch.from_numpy(z["in_xyz"]), out=out, scene_max=float(z["scene_range_max"]),
                skip_weight=float(z["skip_weight"]))
