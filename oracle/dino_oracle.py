"""CPU restatement (plain torch, fp32 or fp64) of the DINOv2 image conditioner: FrozenDinov2ImageEmbedder's
preprocess and the ViT-L/14-reg4 forward behind it.

TEST INFRASTRUCTURE ONLY (checker for tests/ and tools/).  PARITY UNPINNED: there is no golden produced by the
reference's own code (kornia and the hub model are not installed here), so this is a restatement of the contract:

  preprocess   /root/reference/sgm/modules/encoders/modules.py:862-875: kornia resize to (518, 518), bicubic,
               align_corners=True, antialias=True; then (x + 1) / 2; then (x - mean) / std, ImageNet mean / std
  encoder      DINOv2 ViT-L/14 with 4 registers (torch.hub dinov2_vitl14_reg); block loop and output split as the
               reference restates them at modules.py:1321-1362
  embedder     modules.py:907-930 (output_cls=True: (patch tokens, cls token))

[UPSTREAM-MEMORY] kornia.geometry.resize, from memory of kornia's source: an input already at the target size is
returned unchanged; otherwise, when max(H / 518, W / 518) > 1, a separable Gaussian blur runs first with
sigma_i = max((factor_i - 1) / 2, 0.001) and ks_i = int(max(4 sigma_i, 3)) bumped to odd, normalised
exp(-x^2 / 2 sigma^2) on x = arange(ks) - ks // 2, 'reflect' borders, along x then along y; then
F.interpolate(mode="bicubic", align_corners=True).
[UPSTREAM-MEMORY] DINOv2 token preparation: x = cat(cls_token, patches) + pos_embed (used as stored at 518^2), then
the 4 register tokens are inserted after cls without a positional embedding; LayerNorm eps 1e-6; qkv with bias,
"(K H D)" columns, 16 heads of 64, no q/k norm, softmax scale 1/8; MLP fc1 -> exact (erf) GELU -> fc2; LayerScale
gammas ls1, ls2.

emulate_bf16=True rounds the tensor-core operands the way the CUDA path does (weights, the patch matrix, the LayerNorm
outputs, Q / K / V, the unnormalised softmax numerator P, the attention output and the GELU output), like
oracle/dit_oracle.py.
"""
import math

import torch
import torch.nn.functional as F

MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)
IMG_SIZE, PATCH, N_REG, HEADS = 518, 14, 4, 16
EPS = 1e-6

_EMU = False


def _r(x):
    return x.to(torch.bfloat16).to(x.dtype) if _EMU else x


# ---------------------------------------------------------------------------------------------------------------------
# preprocess
# ---------------------------------------------------------------------------------------------------------------------
def blur_params(n, size):
    """(sigma, kernel size) of the antialias blur along an axis of n pixels resized to `size`."""
    sigma = max((n / size - 1.0) / 2.0, 0.001)
    ks = int(max(4.0 * sigma, 3.0))
    return sigma, ks + 1 if ks % 2 == 0 else ks


def gaussian_taps(ks, sigma, dtype):
    x = torch.arange(ks, dtype=dtype) - ks // 2
    s = torch.tensor(sigma, dtype=dtype)
    g = torch.exp(-x.pow(2) / (2 * s.pow(2)))
    return g / g.sum()


def gaussian_blur(x, ks_yx, sigma_yx):
    B, C, H, W = x.shape
    (ky, kx), (sy, sx) = ks_yx, sigma_yx
    y = x.reshape(B * C, 1, H, W)
    y = F.conv2d(F.pad(y, (kx // 2, kx // 2, 0, 0), mode="reflect"), gaussian_taps(kx, sx, x.dtype).view(1, 1, 1, kx))
    y = F.conv2d(F.pad(y, (0, 0, ky // 2, ky // 2), mode="reflect"), gaussian_taps(ky, sy, x.dtype).view(1, 1, ky, 1))
    return y.reshape(B, C, H, W)


def resize(x, size=IMG_SIZE):
    H, W = x.shape[-2:]
    if (H, W) == (size, size):
        return x
    if max(H / size, W / size) > 1:
        (sy, ky), (sx, kx) = blur_params(H, size), blur_params(W, size)
        x = gaussian_blur(x, (ky, kx), (sy, sx))
    return F.interpolate(x, size=(size, size), mode="bicubic", align_corners=True)


def preprocess(img, size=IMG_SIZE, dtype=torch.float32):
    """img [B, 3, H, W] in [-1, 1] -> normalised [B, 3, size, size] in `dtype` (the CUDA path runs it in fp32)."""
    x = resize(img.to(dtype), size)
    x = (x + 1.0) / 2.0
    mean = torch.tensor(MEAN, dtype=torch.float32).to(dtype).view(1, 3, 1, 1)
    std = torch.tensor(STD, dtype=torch.float32).to(dtype).view(1, 3, 1, 1)
    return (x - mean) / std


def patch_matrix(x, patch=PATCH, k_pitch=640):
    """Preprocessed [B, 3, S, S] -> the im2col matrix [B * (S/p)^2, k_pitch] (column c*p*p + ky*p + kx, zero padded)."""
    B, C, S, _ = x.shape
    n = S // patch
    m = x.reshape(B, C, n, patch, n, patch).permute(0, 2, 4, 1, 3, 5).reshape(B * n * n, C * patch * patch)
    return F.pad(m, (0, k_pitch - m.shape[1]))


# ---------------------------------------------------------------------------------------------------------------------
# encoder
# ---------------------------------------------------------------------------------------------------------------------
def _ln(x, sd, p):
    return F.layer_norm(x, x.shape[-1:], sd[p + ".weight"], sd[p + ".bias"], EPS)


def tokens(sd, x):
    """Preprocessed image -> the residual stream [B, 1 + 4 + n^2, D] before block 0."""
    B = x.shape[0]
    w = sd["patch_embed.proj.weight"]
    D = w.shape[0]
    pm = _r(patch_matrix(x, w.shape[-1], w[0].numel()))
    pe = pm @ _r(w.reshape(D, -1)).T + sd["patch_embed.proj.bias"]
    pe = pe.reshape(B, -1, D)
    t = torch.cat([sd["cls_token"].expand(B, -1, -1), pe], 1) + sd["pos_embed"]
    return torch.cat([t[:, :1], sd["register_tokens"].expand(B, -1, -1), t[:, 1:]], 1)


def _qkv(sd, p, x):
    B, N, D = x.shape
    h = _r(_ln(x, sd, p + "norm1"))
    qkv = h @ _r(sd[p + "attn.qkv.weight"]).T + sd[p + "attn.qkv.bias"]
    qkv = qkv.reshape(B, N, 3, HEADS, D // HEADS).permute(2, 0, 3, 1, 4)          # K B H N d
    return _r(qkv[0]), _r(qkv[1]), _r(qkv[2])


def attention(q, k, v):
    scale = 1.0 / math.sqrt(q.shape[-1])
    if not _EMU:
        return torch.softmax((q @ k.transpose(-1, -2)) * scale, -1) @ v
    s = (q @ k.transpose(-1, -2)) * scale
    p = torch.exp(s - s.max(-1, keepdim=True).values)
    return (_r(p) @ v) / p.sum(-1, keepdim=True)                                    # unnormalised P is the MMA operand


def block_forward(sd, p, x):
    B, N, D = x.shape
    q, k, v = _qkv(sd, p, x)
    a = _r(attention(q, k, v).transpose(1, 2).reshape(B, N, D))
    x = x + sd[p + "ls1.gamma"] * (a @ _r(sd[p + "attn.proj.weight"]).T + sd[p + "attn.proj.bias"])
    h = _r(_ln(x, sd, p + "norm2"))
    f = _r(F.gelu(h @ _r(sd[p + "mlp.fc1.weight"]).T + sd[p + "mlp.fc1.bias"]))
    return x + sd[p + "ls2.gamma"] * (f @ _r(sd[p + "mlp.fc2.weight"]).T + sd[p + "mlp.fc2.bias"])


def depth_of(sd):
    return 1 + max(int(k.split(".")[1]) for k in sd if k.startswith("blocks."))


def forward(sd, img, emulate_bf16=False, return_acts=False, dtype=torch.float32):
    """img [B, 3, H, W] in [-1, 1] -> {"x_norm_clstoken" [B, D], "x_norm_patchtokens" [B, n^2, D]} computed in `dtype`
    (state dict cast to it).  return_acts: also the residual stream after every block (list)."""
    global _EMU
    prev, _EMU = _EMU, bool(emulate_bf16)
    try:
        sd = {k: v.to(dtype) for k, v in sd.items()}
        x = tokens(sd, preprocess(img, dtype=dtype))
        acts = []
        for i in range(depth_of(sd)):
            x = block_forward(sd, "blocks.%d." % i, x)
            acts.append(x)
        xn = _ln(x, sd, "norm")
        out = {"x_norm_clstoken": xn[:, 0], "x_norm_patchtokens": xn[:, 1 + N_REG:]}
        if return_acts:
            out["acts"] = acts
        return out
    finally:
        _EMU = prev


def block0_attention_entropy(sd, img, dtype=torch.float32):
    """Mean over batch, heads and queries of the entropy (nats) of block 0's attention rows."""
    sd = {k: v.to(dtype) for k, v in sd.items()}
    x = tokens(sd, preprocess(img, dtype=dtype))
    q, k, _ = _qkv(sd, "blocks.0.", x)
    p = torch.softmax((q @ k.transpose(-1, -2)) / math.sqrt(q.shape[-1]), -1)
    return float(-(p * torch.log(p.clamp_min(1e-30))).sum(-1).mean())


def embedder_forward(sd, img, emulate_bf16=False):
    """FrozenDinov2ImageEmbedder(output_cls=True).forward without dropout: (tokens, z) in img.dtype."""
    o = forward(sd, img, emulate_bf16=emulate_bf16)
    return o["x_norm_patchtokens"].to(img.dtype), o["x_norm_clstoken"].to(img.dtype)
