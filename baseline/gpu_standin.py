"""GPU comparison baselines ("stand-ins") for bench.py -- NOT the product path.

The reference's own GPU build cannot run here: its kernels live in xformers 0.0.22 / diff-surfel-rasterization, which
are neither vendored nor in the offline wheelhouse (BASELINE.md section 4).  north_star's target is stated against
"the reference GPU build", so bench.py times, on the same GPU and the same shapes, what that build does
algorithmically with the libraries this image does have:

  TorchDiT -- the deployed DiT block stack restated as plain PyTorch modules run the way the reference runs them:
      nn.Linear under bf16 autocast (cuBLAS), attention through flash_attn_func (the xformers
      memory_efficient_attention stand-in), separate RMSNorm / modulate / GELU / residual kernels, context K/V
      re-projected in every block on every NFE (SURVEY F11), one 2B forward per NFE for CFG.
      Follows /root/reference/dit/dit_models_xformers.py:765-787 (block), dit/dit_i23d.py:511-567 (forward),
      vit/vision_transformer.py:177-303 (self attention), ldm/modules/attention.py:484-561 (cross attention).

Nothing under gaussiananything_b200/ imports this file.
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F


def _attention(q, k, v):
    """q [B,N,H,d], k/v [B,M,H,d] bf16 -> [B,N,H,d]."""
    try:
        from flash_attn import flash_attn_func
        return flash_attn_func(q, k, v)
    except Exception:
        o = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2))
        return o.transpose(1, 2)


class RMSNorm(nn.Module):                     # /root/reference/dit/norm.py:27-40
    def __init__(self, dim, eps=1e-5):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(dim))
        self.eps = eps

    def forward(self, x):
        y = x.float()
        y = y * torch.rsqrt(y.pow(2).mean(-1, keepdim=True) + self.eps)
        return (y * self.weight).type_as(x)


class Block(nn.Module):
    def __init__(self, D, H, Dc):
        super().__init__()
        self.H = H
        self.scale_shift_table = nn.Parameter(torch.randn(6, D) / D ** 0.5)
        self.norm1, self.norm2, self.prenorm_ca = RMSNorm(D), RMSNorm(D), RMSNorm(D)
        self.qkv, self.proj = nn.Linear(D, 3 * D), nn.Linear(D, D)
        self.q_norm, self.k_norm = RMSNorm(D // H), RMSNorm(D // H)
        self.fc1, self.fc2 = nn.Linear(D, 4 * D), nn.Linear(4 * D, D)
        self.to_q, self.to_k, self.to_v = nn.Linear(D, D, bias=False), nn.Linear(Dc, D, bias=False), nn.Linear(Dc, D, bias=False)
        self.ca_q_norm, self.ca_k_norm = RMSNorm(D // H), RMSNorm(D // H)
        self.to_out = nn.Linear(D, D)

    def forward(self, x, t0, ctx):
        B, N, D = x.shape
        H = self.H
        s_msa, c_msa, g_msa, s_mlp, c_mlp, g_mlp = (self.scale_shift_table[None] + t0.reshape(B, 6, -1)).chunk(6, dim=1)
        h = self.prenorm_ca(x)
        q = self.ca_q_norm(self.to_q(h).view(B, N, H, -1))
        k = self.ca_k_norm(self.to_k(ctx).view(B, ctx.shape[1], H, -1))
        v = self.to_v(ctx).view(B, ctx.shape[1], H, -1)
        x = x + self.to_out(_attention(q.bfloat16(), k.bfloat16(), v.bfloat16()).reshape(B, N, D))
        h = self.norm1(x) * (1 + c_msa) + s_msa
        qkv = self.qkv(h).view(B, N, 3, H, -1)
        q, k, v = self.q_norm(qkv[:, :, 0]), self.k_norm(qkv[:, :, 1]), qkv[:, :, 2]
        x = x + g_msa * self.proj(_attention(q.bfloat16(), k.bfloat16(), v.bfloat16()).reshape(B, N, D))
        h = self.norm2(x) * (1 + c_mlp) + s_mlp
        return x + g_mlp * self.fc2(F.gelu(self.fc1(h)))


class TorchDiT(nn.Module):
    def __init__(self, depth, D, H, Cin, Dc=1024):
        super().__init__()
        self.D, self.Cin = D, Cin
        self.x_fc1, self.x_fc2 = nn.Linear(Cin, D), nn.Linear(D, D)
        self.t_fc1, self.t_fc2 = nn.Linear(256, D), nn.Linear(D, D)
        self.vec_ln, self.vec_fc = nn.LayerNorm(Dc), nn.Linear(Dc, D)
        self.ada = nn.Linear(D, 6 * D)
        self.blocks = nn.ModuleList([Block(D, H, Dc) for _ in range(depth)])
        self.final_table = nn.Parameter(torch.randn(2, D) / D ** 0.5)
        self.final = nn.Linear(D, Cin)

    def forward(self, x, t, ctx, vec):
        half = 128
        freqs = torch.exp(-math.log(10000.0) * torch.arange(half, device=x.device, dtype=torch.float32) / half)
        args = t[:, None].float() * freqs[None]
        temb = self.t_fc2(F.silu(self.t_fc1(torch.cat([torch.cos(args), torch.sin(args)], -1))))
        tt = temb + self.vec_fc(self.vec_ln(vec))
        t0 = self.ada(F.silu(tt))
        h = self.x_fc2(F.gelu(self.x_fc1(x), approximate="tanh"))
        for b in self.blocks:
            h = b(h, t0, ctx)
        shift, scale = (self.final_table[None] + tt[:, None]).chunk(2, dim=1)
        y = F.layer_norm(h.float(), h.shape[-1:], None, None, 1e-6) * (1 + scale) + shift
        return self.final(y).float()

    def forward_with_cfg(self, x, t, ctx, vec, s):
        eps = self.forward(x, t, ctx, vec)
        c, u = eps.chunk(2, 0)
        hlf = u + s * (c - u)
        return torch.cat([hlf, hlf], 0)


def time_torch_dit(dev, depth, D, H, N, Cin=3, M=1369, Dc=1024, nfe=20):
    """ms per NFE (2B = 2 rows: one sample with CFG) of the unfused stand-in: eager and replayed from a CUDA graph."""
    torch.manual_seed(0)
    m = TorchDiT(depth, D, H, Cin, Dc).to(dev).eval()
    x = torch.randn(2, N, Cin, device=dev)
    t = torch.full((2,), 0.3, device=dev)
    ctx = torch.randn(2, M, Dc, device=dev)
    vec = torch.randn(2, Dc, device=dev)
    out = {}
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        for _ in range(3):
            y = m.forward_with_cfg(x, t, ctx, vec, 4.0)
        assert torch.isfinite(y).all()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(dev)
        e0.record()
        for _ in range(nfe):
            m.forward_with_cfg(x, t, ctx, vec, 4.0)
        e1.record()
        e1.synchronize()
        out["eager_ms_per_nfe"] = e0.elapsed_time(e1) / nfe
        try:
            g = torch.cuda.CUDAGraph()
            s = torch.cuda.Stream(dev)
            s.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(s):
                m.forward_with_cfg(x, t, ctx, vec, 4.0)
            torch.cuda.current_stream(dev).wait_stream(s)
            with torch.cuda.graph(g):
                yg = m.forward_with_cfg(x, t, ctx, vec, 4.0)
            for _ in range(3):
                g.replay()
            torch.cuda.synchronize(dev)
            e0.record()
            for _ in range(nfe):
                g.replay()
            e1.record()
            e1.synchronize()
            assert torch.isfinite(yg).all()
            out["graph_ms_per_nfe"] = e0.elapsed_time(e1) / nfe
        except Exception as ex:                              # flash-attn builds that cannot be captured
            out["graph_error"] = repr(ex)
    del m
    torch.cuda.empty_cache()
    return out
