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


# ---------------------------------------------------------------------------------------------------------------------
# TorchDino -- the DINOv2 ViT-L/14-reg4 image conditioner restated as plain PyTorch and run the way the reference runs
# it: nn.Linear / Conv2d under bf16 autocast (cuBLAS / cuDNN), F.scaled_dot_product_attention, separate LayerNorm /
# GELU / LayerScale / residual kernels.  Same state dict layout as gaussiananything_b200.dino (torch.hub layout);
# the image is already 518^2, so the preprocess is the normalisation only.
# ---------------------------------------------------------------------------------------------------------------------
class TorchDino(nn.Module):
    def __init__(self, sd, heads=16):
        super().__init__()
        self.sd = {k: v.float() for k, v in sd.items()}
        self.heads = heads
        self.depth = 1 + max(int(k.split(".")[1]) for k in sd if k.startswith("blocks."))
        self.register_buffer("mean", torch.tensor((0.485, 0.456, 0.406)).view(1, 3, 1, 1))
        self.register_buffer("std", torch.tensor((0.229, 0.224, 0.225)).view(1, 3, 1, 1))

    def to(self, dev):
        self.sd = {k: v.to(dev) for k, v in self.sd.items()}
        return super().to(dev)

    def forward(self, img):
        sd, H = self.sd, self.heads
        x = ((img.float() + 1.0) / 2.0 - self.mean) / self.std
        x = F.conv2d(x, sd["patch_embed.proj.weight"], sd["patch_embed.proj.bias"], stride=14).flatten(2).transpose(1, 2)
        B, _, D = x.shape
        x = torch.cat([sd["cls_token"].expand(B, -1, -1), x], 1) + sd["pos_embed"]
        x = torch.cat([x[:, :1], sd["register_tokens"].expand(B, -1, -1), x[:, 1:]], 1).float()
        N = x.shape[1]
        for i in range(self.depth):
            p = "blocks.%d." % i
            h = F.layer_norm(x, (D,), sd[p + "norm1.weight"], sd[p + "norm1.bias"], 1e-6)
            qkv = F.linear(h, sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"]).view(B, N, 3, H, D // H).permute(2, 0, 3, 1, 4)
            a = F.scaled_dot_product_attention(qkv[0], qkv[1], qkv[2]).transpose(1, 2).reshape(B, N, D)
            x = x + sd[p + "ls1.gamma"] * F.linear(a, sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"])
            h = F.layer_norm(x, (D,), sd[p + "norm2.weight"], sd[p + "norm2.bias"], 1e-6)
            f = F.gelu(F.linear(h, sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"]))
            x = x + sd[p + "ls2.gamma"] * F.linear(f, sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"])
        xn = F.layer_norm(x.float(), (D,), sd["norm.weight"], sd["norm.bias"], 1e-6)
        return {"x_norm_clstoken": xn[:, 0], "x_norm_patchtokens": xn[:, 5:]}


def time_torch_dino(dev, sd, B, min_seconds=2.0):
    """ms per image of TorchDino at batch B (eager, bf16 autocast), device events over >= min_seconds of work."""
    m = TorchDino(sd).to(dev).eval()
    img = torch.rand(B, 3, 518, 518, device=dev) * 2 - 1
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        for _ in range(3):
            y = m(img)
        assert torch.isfinite(y["x_norm_patchtokens"]).all()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(dev)
        e0.record()
        m(img)
        e1.record()
        e1.synchronize()
        reps = max(3, math.ceil(min_seconds / max(e0.elapsed_time(e1) * 1e-3, 1e-6)))
        e0.record()
        for _ in range(reps):
            m(img)
        e1.record()
        e1.synchronize()
    ms = e0.elapsed_time(e1) / reps
    del m
    torch.cuda.empty_cache()
    return {"batch": B, "reps": reps, "ms_per_batch": ms, "ms_per_image": ms / B}


class TorchVaeEncoder:
    """Unfused bf16 PyTorch stand-in of the 3D VAE encoder (HybridEncoderPCDStructuredLatentSNoPCD + posterior) with
    the reference's own op sequence: cuDNN convs and nn.Linear under bf16 autocast, F.group_norm / F.layer_norm,
    F.scaled_dot_product_attention, a loop-per-point farthest-point sampling.  For timing beside
    gaussiananything_b200.vae_encoder.SurfelEncoder (tools/vae_encoder_leg.py), not a checker."""

    def __init__(self, sd, num_frames=8, latent_num=768, device="cuda:0"):
        self.sd = {k: v.to(device).float() for k, v in sd.items()}
        self.V, self.K = num_frames, latent_num

    def _gn(self, x, p, silu=True):
        y = F.group_norm(x.float(), 32, self.sd[p + "weight"], self.sd[p + "bias"], 1e-6)
        return y * torch.sigmoid(y) if silu else y

    def _conv(self, x, p, stride=1):
        sd = self.sd
        if stride == 2:
            return F.conv2d(F.pad(x, (0, 1, 0, 1)), sd[p + "weight"], sd[p + "bias"], stride=2)
        return F.conv2d(x, sd[p + "weight"], sd[p + "bias"], padding=sd[p + "weight"].shape[-1] // 2)

    def _res(self, p, x):
        h = self._conv(self._gn(x, p + "norm1."), p + "conv1.")
        h = self._conv(self._gn(h, p + "norm2."), p + "conv2.")
        if p + "nin_shortcut.weight" in self.sd:
            x = self._conv(x, p + "nin_shortcut.")
        return x + h

    def _ln(self, x, p):
        return F.layer_norm(x.float(), (x.shape[-1],), self.sd[p + "weight"], self.sd[p + "bias"], 1e-5)

    def _mha(self, p, x, ctx, heads, qk_norm=False):
        sd = self.sd
        q, k, v = (F.linear(t, sd[p + n + ".weight"]) for t, n in ((x, "to_q"), (ctx, "to_k"), (ctx, "to_v")))
        B, Nq, C = q.shape
        q, k, v = (t.view(B, -1, heads, C // heads).transpose(1, 2) for t in (q, k, v))
        if qk_norm:
            rms = lambda t, w: (t.float() * torch.rsqrt(t.float().pow(2).mean(-1, keepdim=True) + 1e-5) * w).to(t.dtype)
            q, k = rms(q, sd[p + "q_norm.weight"]), rms(k, sd[p + "k_norm.weight"])
        o = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, Nq, C)
        return F.linear(o, sd[p + "to_out.0.weight"], sd[p + "to_out.0.bias"])

    @staticmethod
    def _fps(pcd, K, start):
        B, N, _ = pcd.shape
        idx = torch.empty(B, K, dtype=torch.long, device=pcd.device)
        md = torch.full((B, N), float("inf"), device=pcd.device)
        cur = start.to(pcd.device).long()
        ar = torch.arange(B, device=pcd.device)
        for k in range(K):
            idx[:, k] = cur
            d = ((pcd - pcd[ar, cur][:, None]) ** 2).sum(-1)
            md = torch.minimum(md, d)
            cur = md.argmax(1)
        return torch.gather(pcd, 1, idx[..., None].expand(B, K, 3))

    def _pe(self, xyz):
        out = [xyz] + [f(xyz * 2.0 ** i) for i in range(10) for f in (torch.sin, torch.cos)]
        p = "encoder.xyz_pos_embed.xyz_projection."
        return F.linear(torch.cat(out, -1), self.sd[p + "weight"], self.sd[p + "bias"])

    @torch.no_grad()
    def encode(self, img, pcd, start):
        sd, V, e = self.sd, self.V, "encoder."
        with torch.autocast("cuda", dtype=torch.bfloat16):
            h = self._conv(img, e + "conv_in.")
            lvl = 0
            while e + "down.%d.block.0.norm1.weight" % lvl in sd:
                h = self._res(e + "down.%d.block.0." % lvl, h)
                if e + "down.%d.downsample.conv.weight" % lvl in sd:
                    h = self._conv(h, e + "down.%d.downsample.conv." % lvl, 2)
                lvl += 1
            h = self._res(e + "mid.block_1.", h)
            a, b = e + "mid.attn_1.", e + "mid.attn_1.transformer_blocks.0."
            n, C, Hf, Wf = h.shape
            x_in = h
            t = self._conv(self._gn(h, a + "norm.", False), a + "proj_in.").flatten(2).transpose(1, 2)
            L = Hf * Wf
            tm = t.reshape(n // V, V * L, -1)
            tn = self._ln(tm, b + "norm1.")
            tm = self._mha(b + "attn1.", tn, tn, 8) + tm
            t = tm.reshape(n, L, -1)
            tn = self._ln(t, b + "norm2.")
            t = self._mha(b + "attn2.", tn, tn, 8) + t
            xg, gate = F.linear(self._ln(t, b + "norm3."), sd[b + "ff.net.0.proj.weight"], sd[b + "ff.net.0.proj.bias"]).chunk(2, -1)
            t = F.linear(xg * F.gelu(gate), sd[b + "ff.net.2.weight"], sd[b + "ff.net.2.bias"]) + t
            h = self._conv(t.transpose(1, 2).reshape(n, -1, Hf, Wf), a + "proj_out.") + x_in
            h = self._gn(self._res(e + "mid.block_2.", h), e + "norm_out.")
            B = n // V
            xyz = img[:, -3:, 4::8, 4::8].reshape(B, V, 3, -1).permute(0, 1, 3, 2).reshape(B, -1, 3)
            tok = h.reshape(B, V, C, L).permute(0, 1, 3, 2).reshape(B, -1, C) + self._pe(xyz)
            qxyz = self._fps(pcd.float(), self.K, start)
            x = self._mha(e + "agg_ca.", self._pe(qxyz), tok, 8, qk_norm=True)
            l = 0
            while e + "srt.transformer.layers.%d.0.norm.weight" % l in sd:
                p = e + "srt.transformer.layers.%d." % l
                hn = self._ln(x, p + "0.norm.")
                qkv = F.linear(hn, sd[p + "0.fn.qkv.weight"], sd[p + "0.fn.qkv.bias"]).view(B, self.K, 3, 8, C // 8)
                q, k, v = qkv.permute(2, 0, 3, 1, 4)
                rms = lambda t, w: (t.float() * torch.rsqrt(t.float().pow(2).mean(-1, keepdim=True) + 1e-5) * w).to(t.dtype)
                q, k = rms(q, sd[p + "0.fn.q_norm.weight"]), rms(k, sd[p + "0.fn.k_norm.weight"])
                o = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, self.K, C)
                x = x + F.linear(o, sd[p + "0.fn.proj.weight"], sd[p + "0.fn.proj.bias"])
                f = F.gelu(F.linear(self._ln(x, p + "1.norm."), sd[p + "1.fn.mlp.0.weight"]) + sd[p + "1.fn.mlp.1.bias"])
                x = x + F.linear(f, sd[p + "1.fn.mlp.2.weight"]) + sd[p + "1.fn.mlp.3.bias"]
                l += 1
            m = "encoder.Mlp_out."
            hh = F.gelu(F.linear(self._ln(x, m + "norm."), sd[m + "fn.fc1.weight"], sd[m + "fn.fc1.bias"]), approximate="tanh")
            hh = F.linear(hh, sd[m + "fn.fc2.weight"], sd[m + "fn.fc2.bias"]).float()
        q = "decoder.superresolution.quant_conv."
        mo = F.linear(F.gelu(F.linear(hh, sd[q + "fc1.weight"], sd[q + "fc1.bias"]), approximate="tanh"),
                      sd[q + "fc2.weight"], sd[q + "fc2.bias"])
        mean, logvar = mo.chunk(2, -1)
        logvar = torch.tanh(logvar / 20.0) * 20.0
        return {"h": hh, "query_pcd_xyz": qxyz, "mean": mean, "logvar": logvar, "std": torch.exp(0.5 * logvar)}
