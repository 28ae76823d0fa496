"""CPU restatement (plain torch, fp32) of the 3D VAE encoder HybridEncoderPCDStructuredLatentSNoPCD and the posterior
the AE applies after it.

TEST INFRASTRUCTURE ONLY (checker for tests/ and tools/).  Pinned against the reference's own classes by
tests/golden/vae_encoder_small.npz (tests/golden/make_vae_encoder_golden.py).

  SD conv encoder      /root/reference/ldm/modules/diffusionmodules/model.py:81-162,469-572 (conv_out = Identity)
  mid.attn_1           /root/reference/ldm/modules/attention.py:706-779 (SpatialTransformer3D, 8 heads x 64;
                       attn1 over all views' tokens, attn2 per view, GEGLU FFN)
  readout              /root/reference/nsr/srt/encoder.py:549-610 (XYZPosEmbed on the 4::8 token xyz, FPS, agg_ca with
                       per-head RMSNorm q/k and no residual, 3 SRT blocks of 8 heads x 32, Mlp_out)
  posterior            /root/reference/vit/vit_triplane.py:1347-1385 (quant_conv, soft-clamped logvar)

Farthest-point sampling follows the kernel's stated rule: distances fp32 (dx*dx + dy*dy) + dz*dz, each operation
rounded on its own, running minimum, ties to the lowest index, the start index passed in.

emulate_bf16=True rounds the tensor-core operands the way the CUDA path does: conv / linear inputs and weights,
Q / K / V, the attention output and the hidden activations of the FFNs.  Norms, residual streams, the readout head
and the posterior stay fp32.
"""
import math

import torch
import torch.nn.functional as F

_EMU = False
GN_EPS, LN_EPS, RMS_EPS = 1e-6, 1e-5, 1e-5


def _r(x):
    return x.to(torch.bfloat16).float() if _EMU else x


def _lin(x, w, b=None):
    y = _r(x) @ _r(w).t()
    return y + b if b is not None else y


def _conv(x, w, b, stride):
    """x [n, C, H, W]; stride 1 pads 1 all round, stride 2 pads (0, 1, 0, 1) (the SD Downsample)."""
    if stride == 2:
        x = F.pad(x, (0, 1, 0, 1))
        return F.conv2d(_r(x), _r(w), b, stride=2)
    return F.conv2d(_r(x), _r(w), b, padding=w.shape[-1] // 2)


def _gn(x, w, b, silu):
    y = F.group_norm(x, 32, w, b, GN_EPS)
    return y * torch.sigmoid(y) if silu else y


def _attn(q, k, v, scale):
    """q [B, H, Nq, d], k / v [B, H, Nk, d] -> [B, Nq, H*d]"""
    q, k, v = _r(q), _r(k), _r(v)
    p = torch.softmax((q @ k.transpose(-1, -2)) * scale, -1)
    o = _r(p @ v)
    B, H, N, d = o.shape
    return o.permute(0, 2, 1, 3).reshape(B, N, H * d)


def _split(t, H):
    B, N, C = t.shape
    return t.reshape(B, N, H, C // H).permute(0, 2, 1, 3)


def _rms(x, w):
    return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + RMS_EPS) * w


def _resblock(sd, p, x):
    h = _conv(_gn(x, sd[p + "norm1.weight"], sd[p + "norm1.bias"], True), sd[p + "conv1.weight"], sd[p + "conv1.bias"], 1)
    h = _conv(_gn(h, sd[p + "norm2.weight"], sd[p + "norm2.bias"], True), sd[p + "conv2.weight"], sd[p + "conv2.bias"], 1)
    if p + "nin_shortcut.weight" in sd:
        w = sd[p + "nin_shortcut.weight"]
        x = F.conv2d(_r(x), _r(w), sd[p + "nin_shortcut.bias"])
    return x + h


def _mha(sd, p, x, ctx, heads, q_norm=False):
    q, k, v = _lin(x, sd[p + "to_q.weight"]), _lin(ctx, sd[p + "to_k.weight"]), _lin(ctx, sd[p + "to_v.weight"])
    q, k, v = _split(q, heads), _split(k, heads), _split(v, heads)
    if q_norm:
        q, k = _rms(q, sd[p + "q_norm.weight"]), _rms(k, sd[p + "k_norm.weight"])
    o = _attn(q, k, v, 1.0 / math.sqrt(q.shape[-1]))
    return _lin(o, sd[p + "to_out.0.weight"], sd[p + "to_out.0.bias"])


def _ln(x, sd, p):
    return F.layer_norm(x, (x.shape[-1],), sd[p + "weight"], sd[p + "bias"], LN_EPS)


def spatial_transformer_3d(sd, p, x, num_frames, heads=8):
    n, C, H, W = x.shape
    x_in = x
    h = _gn(x, sd[p + "norm.weight"], sd[p + "norm.bias"], False)
    h = F.conv2d(_r(h), _r(sd[p + "proj_in.weight"]), sd[p + "proj_in.bias"])
    t = h.flatten(2).transpose(1, 2)                                   # [n, HW, inner]
    b = p + "transformer_blocks.0."
    B = n // num_frames
    L = H * W
    tm = t.reshape(B, num_frames * L, -1)
    tm = _mha(sd, b + "attn1.", _ln(tm, sd, b + "norm1."), _ln(tm, sd, b + "norm1."), heads) + tm
    t = tm.reshape(n, L, -1)
    t = _mha(sd, b + "attn2.", _ln(t, sd, b + "norm2."), _ln(t, sd, b + "norm2."), heads) + t
    g = _lin(_ln(t, sd, b + "norm3."), sd[b + "ff.net.0.proj.weight"], sd[b + "ff.net.0.proj.bias"])
    xg, gate = g.chunk(2, -1)
    t = _lin(_r(xg * F.gelu(gate)), sd[b + "ff.net.2.weight"], sd[b + "ff.net.2.bias"]) + t
    h = t.transpose(1, 2).reshape(n, -1, H, W)
    h = F.conv2d(_r(h), _r(sd[p + "proj_out.weight"]), sd[p + "proj_out.bias"])
    return h + x_in


def conv_encoder(sd, x, num_frames, acts=None):
    """x [B*V, 15, H, W] -> h [B*V, 256, H/8, W/8] (after norm_out + SiLU); acts collects the per-level outputs."""
    e = "encoder."
    h = _conv(x, sd[e + "conv_in.weight"], sd[e + "conv_in.bias"], 1)
    lvl = 0
    while e + "down.%d.block.0.norm1.weight" % lvl in sd:
        h = _resblock(sd, e + "down.%d.block.0." % lvl, h)
        if acts is not None:
            acts["level%d" % lvl] = h
        if e + "down.%d.downsample.conv.weight" % lvl in sd:
            p = e + "down.%d.downsample.conv." % lvl
            h = _conv(h, sd[p + "weight"], sd[p + "bias"], 2)
        lvl += 1
    h = _resblock(sd, e + "mid.block_1.", h)
    h = spatial_transformer_3d(sd, e + "mid.attn_1.", h, num_frames)
    if acts is not None:
        acts["attn_1"] = h
    h = _resblock(sd, e + "mid.block_2.", h)
    return _gn(h, sd[e + "norm_out.weight"], sd[e + "norm_out.bias"], True)


def posenc(xyz):
    """NeRF encoding, 10 octaves, input included: [..., 3] -> [..., 63]"""
    out = [xyz]
    for i in range(10):
        f = 2.0 ** i
        out += [torch.sin(xyz * f), torch.cos(xyz * f)]
    return torch.cat(out, -1)


def xyz_pos_embed(sd, xyz):
    p = "encoder.xyz_pos_embed.xyz_projection."
    return _lin(posenc(xyz), sd[p + "weight"], sd[p + "bias"])


def fps(pcd, K, start_idx):
    """pcd [B, N, 3] fp32, start_idx [B] -> (xyz [B, K, 3], idx [B, K] int64)"""
    pcd = pcd.float()
    B, N, _ = pcd.shape
    idx = torch.zeros(B, K, dtype=torch.int64)
    for b in range(B):
        P = pcd[b]
        md = torch.full((N,), float("inf"))
        cur = int(start_idx[b])
        for k in range(K):
            idx[b, k] = cur
            if k + 1 == K:
                break
            d = P - P[cur]
            dist = d[:, 0] * d[:, 0]
            dist = dist + d[:, 1] * d[:, 1]
            dist = dist + d[:, 2] * d[:, 2]
            md = torch.minimum(md, dist)
            cur = int(torch.argmax(md))                  # first maximum = lowest index
    xyz = torch.gather(pcd, 1, idx[..., None].expand(B, K, 3))
    return xyz, idx


def _srt_block(sd, p, x, heads=8):
    a = p + "0."
    h = _ln(x, sd, a + "norm.")
    qkv = _lin(h, sd[a + "fn.qkv.weight"], sd[a + "fn.qkv.bias"])
    B, N, C3 = qkv.shape
    C = C3 // 3
    q, k, v = qkv.reshape(B, N, 3, heads, C // heads).permute(2, 0, 3, 1, 4)
    q, k = _rms(_r(q), sd[a + "fn.q_norm.weight"]), _rms(_r(k), sd[a + "fn.k_norm.weight"])
    o = _attn(q, k, v, (C // heads) ** -0.5)
    x = _lin(o, sd[a + "fn.proj.weight"], sd[a + "fn.proj.bias"]) + x
    m = p + "1."
    h = _ln(x, sd, m + "norm.")
    h = _r(F.gelu(_lin(h, sd[m + "fn.mlp.0.weight"]) + sd[m + "fn.mlp.1.bias"]))
    return _lin(h, sd[m + "fn.mlp.2.weight"]) + sd[m + "fn.mlp.3.bias"] + x


def encode(sd, img, pcd, num_frames, K, start_idx, emulate_bf16=False, acts=None):
    """img [B*V, 15, H, W], pcd [B, N, 3] -> {'h' [B, K, 2 zc], 'query_pcd_xyz' [B, K, 3], 'fps_idx' [B, K]}"""
    global _EMU
    _EMU = emulate_bf16
    try:
        img, pcd = img.float(), pcd.float()
        h = conv_encoder(sd, img, num_frames, acts)
        n, C, Hf, Wf = h.shape
        B = n // num_frames
        xyz = img[:, -3:, 4::8, 4::8]
        tok_xyz = xyz.reshape(B, num_frames, 3, -1).permute(0, 1, 3, 2).reshape(B, -1, 3)
        tok = h.reshape(B, num_frames, C, Hf * Wf).permute(0, 1, 3, 2).reshape(B, -1, C)
        tok = tok + xyz_pos_embed(sd, tok_xyz)
        qxyz, idx = fps(pcd, K, start_idx)
        qh = xyz_pos_embed(sd, qxyz)
        x = _mha(sd, "encoder.agg_ca.", qh, tok, 8, q_norm=True)
        if acts is not None:
            acts["agg_ca"] = x
        l = 0
        while "encoder.srt.transformer.layers.%d.0.norm.weight" % l in sd:
            x = _srt_block(sd, "encoder.srt.transformer.layers.%d." % l, x)
            l += 1
        if acts is not None:
            acts["srt"] = x
        _EMU = False                                                 # the readout head runs in fp32
        p = "encoder.Mlp_out."
        hh = F.gelu(_lin(_ln(x, sd, p + "norm."), sd[p + "fn.fc1.weight"], sd[p + "fn.fc1.bias"]), approximate="tanh")
        hh = _lin(hh, sd[p + "fn.fc2.weight"], sd[p + "fn.fc2.bias"])
        return {"h": hh, "query_pcd_xyz": qxyz, "fps_idx": idx}
    finally:
        _EMU = False


def posterior(sd, h, noise=None):
    """quant_conv + DiagonalGaussianDistribution(soft_clamp=True) -> mean, logvar, std, latent ([B, K, zc])"""
    q = "decoder.superresolution.quant_conv."
    m = F.gelu(h @ sd[q + "fc1.weight"].t() + sd[q + "fc1.bias"], approximate="tanh")
    m = m @ sd[q + "fc2.weight"].t() + sd[q + "fc2.bias"]
    mean, logvar = m.chunk(2, -1)
    logvar = torch.tanh(logvar / 20.0) * 20.0
    std = torch.exp(0.5 * logvar)
    latent = mean + std * noise if noise is not None else mean
    return {"mean": mean, "logvar": logvar, "std": std, "latent_normalized": latent}
