"""3D VAE encoder: posed multi-view RGB-D-N renderings -> the point-cloud-structured latent, on the library's kernels.

Mirrors the reference's deployed encoder HybridEncoderPCDStructuredLatentSNoPCD (/root/reference/nsr/srt/encoder.py:
454-652, configuration of shell_scripts/release/inference/vae-3d.sh) and the posterior of
vit.vit_triplane...vae_reparameterization (/root/reference/vit/vit_triplane.py:1347-1385):

  SD conv encoder   3x3 convs: ga_conv3x3_bf16 (implicit GEMM on wgmma); GroupNorm(32)+SiLU: ga_group_norm_nhwc;
                    1x1 nin_shortcut: ga_gemm_bf16_tn (NHWC makes it a plain GEMM)
  mid.attn_1        SpatialTransformer3D: GroupNorm, proj_in / proj_out GEMMs, attn1 over all views' tokens and attn2
                    per view on ga_attention_bf16 (head_dim 64), GEGLU FFN (GA_EPI_GEGLU_BF16)
  readout           token xyz gather + XYZPosEmbed (ga_vae_enc_input, ga_xyz_posenc + GEMM), ga_fps, agg_ca with
                    per-head RMSNorm q / k (GA_EPI_HEADS), 3 SRT blocks of 8 heads x 32 (ga_heads32_split pads the
                    heads to 64 for ga_attention_bf16), Mlp_out + quant_conv + posterior (ga_vae_enc_head, fp32)

Activations are NHWC; bf16 tensor-core operands, fp32 accumulation, fp32 residual streams and norms.  No CPU fallback.
"""
import ctypes as C

import torch

from . import _launch, _lib
from ._launch import epilogue, gemm, ptr as _p, round_up as _round_up
from ._lib import EPI_BF16, EPI_F32, EPI_GEGLU_BF16, EPI_GELU_BF16, EPI_HEADS, EPI_RESID_GATE_F32, GaVaeEncHead


def _expected_keys(ch=64, ch_mult=(1, 2, 4, 4), in_channels=15, z_channels=10, srt_depth=3, heads=8, d_head=64):
    """{key: shape} of the reference AE checkpoint entries the encoder reads (tests/golden/vae_encoder_keys.json
    records the same table from the reference classes)."""
    k = {}
    lin = lambda n, o, i, bias=True: k.update({n + ".weight": (o, i), **({n + ".bias": (o,)} if bias else {})})
    conv = lambda n, o, i, s: k.update({n + ".weight": (o, i, s, s), n + ".bias": (o,)})
    norm = lambda n, c: k.update({n + ".weight": (c,), n + ".bias": (c,)})
    e = "encoder."

    def res(p, ci, co):
        norm(p + "norm1", ci); conv(p + "conv1", co, ci, 3); norm(p + "norm2", co); conv(p + "conv2", co, co, 3)
        if ci != co:
            conv(p + "nin_shortcut", co, ci, 1)

    conv(e + "conv_in", ch, in_channels, 3)
    cin = ch
    for i, m in enumerate(ch_mult):
        res(e + "down.%d.block.0." % i, cin, ch * m)
        cin = ch * m
        if i != len(ch_mult) - 1:
            conv(e + "down.%d.downsample.conv" % i, cin, cin, 3)
    D = cin
    res(e + "mid.block_1.", D, D)
    res(e + "mid.block_2.", D, D)
    a = e + "mid.attn_1."
    inner = heads * d_head
    norm(a + "norm", D); conv(a + "proj_in", inner, D, 1); conv(a + "proj_out", D, inner, 1)
    b = a + "transformer_blocks.0."
    for at in ("attn1.", "attn2."):
        for n in ("to_q", "to_k", "to_v"):
            lin(b + at + n, inner, inner, bias=False)
        lin(b + at + "to_out.0", inner, inner)
    lin(b + "ff.net.0.proj", 8 * inner, inner); lin(b + "ff.net.2", inner, 4 * inner)
    for n in ("norm1", "norm2", "norm3"):
        norm(b + n, inner)
    norm(e + "norm_out", D)
    for l in range(srt_depth):
        t = e + "srt.transformer.layers.%d." % l
        norm(t + "0.norm", D); norm(t + "1.norm", D)
        lin(t + "0.fn.qkv", 3 * D, D); lin(t + "0.fn.proj", D, D)
        k[t + "0.fn.q_norm.weight"] = (D // heads,); k[t + "0.fn.k_norm.weight"] = (D // heads,)
        k[t + "1.fn.mlp.0.weight"] = (4 * D, D); k[t + "1.fn.mlp.1.bias"] = (4 * D,)
        k[t + "1.fn.mlp.2.weight"] = (D, 4 * D); k[t + "1.fn.mlp.3.bias"] = (D,)
    g = e + "agg_ca."
    for n in ("to_q", "to_k", "to_v"):
        lin(g + n, inner, D, bias=False)
    lin(g + "to_out.0", D, inner)
    k[g + "q_norm.weight"] = (d_head,); k[g + "k_norm.weight"] = (d_head,)
    lin(e + "xyz_pos_embed.xyz_projection", D, 63)
    norm(e + "Mlp_out.norm", D)
    lin(e + "Mlp_out.fn.fc1", D, D); lin(e + "Mlp_out.fn.fc2", 2 * z_channels, D)
    q = "decoder.superresolution.quant_conv."
    lin(q + "fc1", 2 * z_channels, 2 * z_channels); lin(q + "fc2", 2 * z_channels, 2 * z_channels)
    return k


def check_state_dict(sd, **cfg):
    """Strict check of the encoder's entries: every expected key present with its shape.  Keys outside the encoder
    (the rest of the AE: decoder.*) are ignored; an unexpected encoder.* key raises, named."""
    want = _expected_keys(**cfg)
    missing = sorted(k for k in want if k not in sd)
    unexpected = sorted(k for k in sd if k.startswith("encoder.") and k not in want)
    bad = sorted(k for k in want if k in sd and tuple(sd[k].shape) != tuple(want[k]))
    if missing or unexpected or bad:
        raise KeyError("SurfelEncoder state_dict: missing %s, unexpected %s, wrong shape %s"
                       % (missing, unexpected, ["%s %s != %s" % (k, tuple(sd[k].shape), want[k]) for k in bad]))


class Posterior:
    """DiagonalGaussianDistribution(soft_clamp=True) over [B, K, zc] (the reference's is [B, zc, K])."""

    def __init__(self, mean, logvar, std):
        self.mean, self.logvar, self.std = mean, logvar, std
        self.var = std * std

    def sample(self, generator=None):
        eps = torch.randn(self.mean.shape, generator=generator).to(self.mean.device)
        return self.mean + self.std * eps

    def mode(self):
        return self.mean


class SurfelEncoder:
    use_graph = _launch.graph_switch()

    def __init__(self, state_dict, num_frames=8, latent_num=768, ch=64, ch_mult=(1, 2, 4, 4), in_channels=15,
                 z_channels=10, device="cuda:0"):
        self.L = _lib.lib()
        self.device = dev = torch.device(device)
        if dev.type != "cuda":
            raise RuntimeError("gaussiananything_b200 needs a CUDA device (no CPU fallback)")
        cfg = dict(ch=ch, ch_mult=tuple(ch_mult), in_channels=in_channels, z_channels=z_channels)
        check_state_dict(state_dict, **cfg)
        self.V, self.K, self.zc, self.cin = int(num_frames), int(latent_num), int(z_channels), int(in_channels)
        self.cin_p = _round_up(self.cin, 8)
        sd = state_dict
        f32 = lambda k: sd[k].detach().to(device=dev, dtype=torch.float32).contiguous()
        b16 = lambda t: t.detach().to(device=dev, dtype=torch.bfloat16).contiguous()
        e = "encoder."

        def conv3(p, cin_p=None):
            w = sd[p + ".weight"].float()
            co, ci = w.shape[:2]
            cp = cin_p or ci
            wp = torch.zeros(co, 3, 3, cp)
            wp[..., :ci] = w.permute(0, 2, 3, 1)
            kp = _round_up(9 * cp, 64)
            out = torch.zeros(co, kp)
            out[:, :9 * cp] = wp.reshape(co, 9 * cp)
            return dict(w=b16(out), b=f32(p + ".bias"), kp=kp, cout=co)

        def res(p):
            r = dict(n1w=f32(p + "norm1.weight"), n1b=f32(p + "norm1.bias"), c1=conv3(p + "conv1"),
                     n2w=f32(p + "norm2.weight"), n2b=f32(p + "norm2.bias"), c2=conv3(p + "conv2"))
            if p + "nin_shortcut.weight" in sd:
                r["nin_w"] = b16(sd[p + "nin_shortcut.weight"][:, :, 0, 0])
                r["nin_b"] = f32(p + "nin_shortcut.bias")
            return r

        self.conv_in = conv3(e + "conv_in", self.cin_p)
        self.levels = []
        for i in range(len(ch_mult)):
            lv = dict(block=res(e + "down.%d.block.0." % i))
            if e + "down.%d.downsample.conv.weight" % i in sd:
                lv["down"] = conv3(e + "down.%d.downsample.conv" % i)
            self.levels.append(lv)
        self.mid1, self.mid2 = res(e + "mid.block_1."), res(e + "mid.block_2.")
        a, b = e + "mid.attn_1.", e + "mid.attn_1.transformer_blocks.0."
        inner = sd[a + "proj_in.weight"].shape[0]
        self.inner, self.D = inner, sd[a + "proj_in.weight"].shape[1]
        ffw, ffb = sd[b + "ff.net.0.proj.weight"].float(), sd[b + "ff.net.0.proj.bias"].float()
        hid = ffw.shape[0] // 2
        # GEGLU: rows interleaved (x_j, gate_j) so that one output tile holds both halves
        ffw_i = torch.stack([ffw[:hid], ffw[hid:]], 1).reshape(2 * hid, -1)
        ffb_i = torch.stack([ffb[:hid], ffb[hid:]], 1).reshape(2 * hid)
        self.mv = dict(gn_w=f32(a + "norm.weight"), gn_b=f32(a + "norm.bias"),
                       pin_w=b16(sd[a + "proj_in.weight"][:, :, 0, 0]), pin_b=f32(a + "proj_in.bias"),
                       pout_w=b16(sd[a + "proj_out.weight"][:, :, 0, 0]), pout_b=f32(a + "proj_out.bias"),
                       ff1_w=b16(ffw_i), ff1_b=ffb_i.to(dev).contiguous(), ff_hid=hid,
                       ff2_w=b16(sd[b + "ff.net.2.weight"]), ff2_b=f32(b + "ff.net.2.bias"))
        for j, at in enumerate(("attn1.", "attn2.")):
            p = b + at
            self.mv["qkv%d" % j] = b16(torch.cat([sd[p + "to_q.weight"], sd[p + "to_k.weight"], sd[p + "to_v.weight"]], 0))
            self.mv["out%d_w" % j], self.mv["out%d_b" % j] = b16(sd[p + "to_out.0.weight"]), f32(p + "to_out.0.bias")
            self.mv["ln%d_w" % j], self.mv["ln%d_b" % j] = f32(b + "norm%d.weight" % (j + 1)), f32(b + "norm%d.bias" % (j + 1))
        self.mv["ln2_w"], self.mv["ln2_b"] = f32(b + "norm3.weight"), f32(b + "norm3.bias")
        self.norm_out = (f32(e + "norm_out.weight"), f32(e + "norm_out.bias"))
        D = self.D
        xw = torch.zeros(D, 64)
        xw[:, :63] = sd[e + "xyz_pos_embed.xyz_projection.weight"].float()
        self.xyz_w, self.xyz_b = b16(xw), f32(e + "xyz_pos_embed.xyz_projection.bias")
        g = e + "agg_ca."
        qn, kn = f32(g + "q_norm.weight"), f32(g + "k_norm.weight")
        self.agg = dict(q_w=b16(sd[g + "to_q.weight"]), kv_w=b16(torch.cat([sd[g + "to_k.weight"], sd[g + "to_v.weight"]], 0)),
                        q_n=qn, k_n=kn, out_w=b16(sd[g + "to_out.0.weight"]), out_b=f32(g + "to_out.0.bias"),
                        bound=8.16 * float(qn.abs().max()) * float(kn.abs().max()))
        self.srt = []
        l = 0
        while e + "srt.transformer.layers.%d.0.norm.weight" % l in sd:
            t = e + "srt.transformer.layers.%d." % l
            hd = sd[t + "0.fn.q_norm.weight"].shape[0]
            nh = D // hd
            assert hd == 32, "the SRT blocks run with head_dim 32"
            pw = sd[t + "0.fn.proj.weight"].float().reshape(D, nh, hd)
            pwp = torch.zeros(D, nh, 64)
            pwp[..., :hd] = pw                                      # attention output is padded to 64 per head
            self.srt.append(dict(n1w=f32(t + "0.norm.weight"), n1b=f32(t + "0.norm.bias"),
                                 qkv_w=b16(sd[t + "0.fn.qkv.weight"]), qkv_b=f32(t + "0.fn.qkv.bias"),
                                 q_n=f32(t + "0.fn.q_norm.weight"), k_n=f32(t + "0.fn.k_norm.weight"), heads=nh,
                                 proj_w=b16(pwp.reshape(D, nh * 64)), proj_b=f32(t + "0.fn.proj.bias"),
                                 n2w=f32(t + "1.norm.weight"), n2b=f32(t + "1.norm.bias"),
                                 w1=b16(sd[t + "1.fn.mlp.0.weight"]), b1=f32(t + "1.fn.mlp.1.bias"),
                                 w2=b16(sd[t + "1.fn.mlp.2.weight"]), b2=f32(t + "1.fn.mlp.3.bias")))
            l += 1
        p, q = e + "Mlp_out.", "decoder.superresolution.quant_conv."
        self.head_t = dict(ln_w=f32(p + "norm.weight"), ln_b=f32(p + "norm.bias"), fc1_w=f32(p + "fn.fc1.weight"),
                           fc1_b=f32(p + "fn.fc1.bias"), fc2_w=f32(p + "fn.fc2.weight"), fc2_b=f32(p + "fn.fc2.bias"),
                           q1_w=f32(q + "fc1.weight"), q1_b=f32(q + "fc1.bias"), q2_w=f32(q + "fc2.weight"),
                           q2_b=f32(q + "fc2.bias"))
        self.head = GaVaeEncHead(**{k: v.data_ptr() for k, v in self.head_t.items()}, ln_eps=1e-5)
        self.head_hid = self.head_t["fc1_w"].shape[0]
        self._graphs = _launch.GraphCache("GA_B200_VAE_ENC_GRAPH")          # (B, V, H, W, N) -> graph

    # ---- launch helpers
    def _conv(self, x, n, H, W, cin, cv, stride, st, residual=None, out_bf16=False, out_f32=True):
        Ho, Wo = self.L.ga_conv3x3_out_size(H, stride), self.L.ga_conv3x3_out_size(W, stride)
        M = n * Ho * Wo
        of = torch.empty(M, cv["cout"], device=self.device) if out_f32 else None
        ob = torch.empty(M, cv["cout"], device=self.device, dtype=torch.bfloat16) if out_bf16 else None
        _lib.check(self.L.ga_conv3x3_bf16(_p(x), n, H, W, cin, _p(cv["w"]), cv["kp"], _p(cv["b"]), cv["cout"], stride,
                                          _p(residual), _p(of), _p(ob), st), "ga_conv3x3_bf16")
        return of, ob, Ho, Wo

    def _gn(self, x, w, b, n, HW, Cc, silu, scratch, st, bf16=True):
        out = torch.empty(n * HW, Cc, device=self.device, dtype=torch.bfloat16 if bf16 else torch.float32)
        _lib.check(self.L.ga_group_norm_nhwc(_p(x), _p(w), _p(b), n, HW, Cc, 1e-6, int(silu), _p(out), int(bf16),
                                             _p(scratch), scratch.numel(), st), "ga_group_norm_nhwc")
        return out

    def _bf16(self, x, st):
        y = torch.empty(x.shape, device=self.device, dtype=torch.bfloat16)
        _lib.check(self.L.ga_f32_to_bf16(_p(x), _p(y), x.numel(), st), "f32_to_bf16")
        return y

    def _resblock(self, r, x, n, H, W, gn_scratch, st):
        """x fp32 NHWC [n*H*W, Cin] -> (fp32, bf16) [n*H*W, Cout]"""
        cin, cout = x.shape[1], r["c1"]["cout"]
        a = self._gn(x, r["n1w"], r["n1b"], n, H * W, cin, True, gn_scratch, st)
        h, _, _, _ = self._conv(a, n, H, W, cin, r["c1"], 1, st)
        a2 = self._gn(h, r["n2w"], r["n2b"], n, H * W, cout, True, gn_scratch, st)
        res = x
        if "nin_w" in r:
            res = torch.empty(n * H * W, cout, device=self.device)
            gemm(self._bf16(x, st), r["nin_w"], n * H * W, cout, cin,
                 epilogue(EPI_F32, bias=r["nin_b"], out=res, ld_out=cout), st)
        of, ob, _, _ = self._conv(a2, n, H, W, cout, r["c2"], 1, st, residual=res, out_bf16=True)
        return of, ob

    def _mha_self(self, hln, R, rows_per_batch, qkv_w, out_w, out_b, resid, st):
        """self-attention of 8 heads x 64 over sequences of rows_per_batch tokens; adds to_out(.) into resid"""
        inner, H = self.inner, self.inner // 64
        nb = R // rows_per_batch
        Np = _round_up(rows_per_batch, 128)
        z = lambda *s: torch.zeros(*s, device=self.device, dtype=torch.bfloat16)
        qb, kb, vt = z(nb * H, Np, 64), z(nb * H, Np, 64), z(nb * H, 64, Np)
        gemm(hln, qkv_w, R, 3 * inner, inner,
             epilogue(EPI_HEADS, q=qb, k=kb, vt=vt, heads=H, first_part=0, tok_pitch=Np,
                      rows_per_batch=rows_per_batch), st)
        ao = torch.empty(R, inner, device=self.device, dtype=torch.bfloat16)
        _lib.check(self.L.ga_attention_bf16(_p(qb), _p(kb), _p(vt), _p(ao), nb, H, rows_per_batch, rows_per_batch, Np, Np,
                                            0.125, 0.0, st), "attention")
        gemm(ao, out_w, R, inner, inner, epilogue(EPI_RESID_GATE_F32, bias=out_b, out=resid, ld_out=inner), st)

    def _attn_1(self, x, n, H, W, gn_scratch, st):
        """SpatialTransformer3D, in place on x (fp32 NHWC [n*H*W, D])"""
        m, D, inner = self.mv, self.D, self.inner
        R, HW = n * H * W, H * W
        g = self._gn(x, m["gn_w"], m["gn_b"], n, HW, D, False, gn_scratch, st)
        t = torch.empty(R, inner, device=self.device)
        gemm(g, m["pin_w"], R, inner, D, epilogue(EPI_F32, bias=m["pin_b"], out=t, ld_out=inner), st)
        hln = torch.empty(R, inner, device=self.device, dtype=torch.bfloat16)
        L = self.L
        for j, rpb in enumerate((self.V * HW, HW)):                 # attn1: all views' tokens; attn2: per view
            _lib.check(L.ga_layernorm_modulate(_p(t), _p(m["ln%d_w" % j]), _p(m["ln%d_b" % j]), None, None, 0, 1, _p(hln),
                                               R, inner, 1e-5, st), "norm%d" % (j + 1))
            self._mha_self(hln, R, rpb, m["qkv%d" % j], m["out%d_w" % j], m["out%d_b" % j], t, st)
        _lib.check(L.ga_layernorm_modulate(_p(t), _p(m["ln2_w"]), _p(m["ln2_b"]), None, None, 0, 1, _p(hln), R, inner, 1e-5,
                                           st), "norm3")
        hid = m["ff_hid"]
        ff = torch.empty(R, hid, device=self.device, dtype=torch.bfloat16)
        gemm(hln, m["ff1_w"], R, 2 * hid, inner, epilogue(EPI_GEGLU_BF16, bias=m["ff1_b"], out=ff, ld_out=hid), st)
        gemm(ff, m["ff2_w"], R, inner, hid, epilogue(EPI_RESID_GATE_F32, bias=m["ff2_b"], out=t, ld_out=inner), st)
        gemm(self._bf16(t, st), m["pout_w"], R, D, inner,
             epilogue(EPI_RESID_GATE_F32, bias=m["pout_b"], out=x, ld_out=D), st)
        return x

    def _launches(self, img, pcd, start_idx, noise, acts=None):
        L, dev, V, K, D = self.L, self.device, self.V, self.K, self.D
        n, cin, H, W = img.shape
        B = n // V
        Np = pcd.shape[1]
        st = _launch.stream(dev)
        gn_scratch = torch.empty(L.ga_group_norm_scratch_bytes(n, H * W), device=dev, dtype=torch.uint8)
        Ht, Wt = (H - 4 + 7) // 8, (W - 4 + 7) // 8
        xin = torch.empty(n * H * W, self.cin_p, device=dev, dtype=torch.bfloat16)
        txyz = torch.empty(n * Ht * Wt, 3, device=dev)
        _lib.check(L.ga_vae_enc_input(_p(img), n, cin, H, W, self.cin_p, _p(xin), cin - 3, 8, 4, _p(txyz), st), "input")
        x, _, _, _ = self._conv(xin, n, H, W, self.cin_p, self.conv_in, 1, st)
        for i, lv in enumerate(self.levels):
            x, xb = self._resblock(lv["block"], x, n, H, W, gn_scratch, st)
            if acts is not None:
                acts["level%d" % i] = (x, H, W)
            if "down" in lv:
                x, _, H, W = self._conv(xb, n, H, W, x.shape[1], lv["down"], 2, st)
        assert H * W == Ht * Wt, "token xyz grid %dx%d does not match the feature map %dx%d" % (Ht, Wt, H, W)
        x, _ = self._resblock(self.mid1, x, n, H, W, gn_scratch, st)
        x = self._attn_1(x, n, H, W, gn_scratch, st)
        if acts is not None:
            acts["attn_1"] = (x.clone(), H, W)
        x, _ = self._resblock(self.mid2, x, n, H, W, gn_scratch, st)
        R = n * H * W
        tok = self._gn(x, self.norm_out[0], self.norm_out[1], n, H * W, D, True, gn_scratch, st, bf16=False)
        # ---- readout: tokens "(B V H W) C" are the NHWC rows as they stand
        pe = torch.empty(R, 64, device=dev, dtype=torch.bfloat16)
        _lib.check(L.ga_xyz_posenc(_p(txyz), _p(pe), R, st), "token posenc")
        gemm(pe, self.xyz_w, R, D, 64, epilogue(EPI_RESID_GATE_F32, bias=self.xyz_b, out=tok, ld_out=D), st)
        qidx = torch.empty(B, K, device=dev, dtype=torch.int32)
        qxyz = torch.empty(B, K, 3, device=dev)
        _lib.check(L.ga_fps(_p(pcd), B, Np, K, _p(start_idx), _p(qidx), _p(qxyz), st), "fps")
        RQ = B * K
        qpe = torch.empty(RQ, 64, device=dev, dtype=torch.bfloat16)
        _lib.check(L.ga_xyz_posenc(_p(qxyz), _p(qpe), RQ, st), "query posenc")
        qh = torch.empty(RQ, D, device=dev, dtype=torch.bfloat16)
        gemm(qpe, self.xyz_w, RQ, D, 64, epilogue(EPI_BF16, bias=self.xyz_b, out=qh, ld_out=D), st)
        a, inner, Hh = self.agg, self.inner, self.inner // 64
        Lk = V * H * W
        PQ, PK = _round_up(K, 128), _round_up(Lk, 128)
        zb = lambda *s: torch.zeros(*s, device=dev, dtype=torch.bfloat16)
        qb, kb, vt = zb(B * Hh, PQ, 64), zb(B * Hh, PK, 64), zb(B * Hh, 64, PK)
        gemm(qh, a["q_w"], RQ, inner, D, epilogue(EPI_HEADS, q=qb, qn_w=a["q_n"], heads=Hh, first_part=0,
                                                   tok_pitch=PQ, rows_per_batch=K), st)
        gemm(self._bf16(tok, st), a["kv_w"], R, 2 * inner, D,
             epilogue(EPI_HEADS, k=kb, vt=vt, kn_w=a["k_n"], heads=Hh, first_part=1, tok_pitch=PK, rows_per_batch=Lk), st)
        ao = torch.empty(RQ, inner, device=dev, dtype=torch.bfloat16)
        _lib.check(L.ga_attention_bf16(_p(qb), _p(kb), _p(vt), _p(ao), B, Hh, K, Lk, PQ, PK, 0.125, a["bound"], st), "agg_ca")
        xs = torch.empty(RQ, D, device=dev)
        gemm(ao, a["out_w"], RQ, D, inner, epilogue(EPI_F32, bias=a["out_b"], out=xs, ld_out=D), st)
        if acts is not None:
            acts["agg_ca"] = xs.clone()
        # ---- SRT blocks (heads of 32, padded to 64 for the attention kernel)
        hs = torch.empty(RQ, D, device=dev, dtype=torch.bfloat16)
        for blk in self.srt:
            nh = blk["heads"]
            qkv = torch.empty(RQ, 3 * D, device=dev, dtype=torch.bfloat16)
            _lib.check(L.ga_layernorm_modulate(_p(xs), _p(blk["n1w"]), _p(blk["n1b"]), None, None, 0, 1, _p(hs), RQ, D, 1e-5,
                                               st), "srt norm1")
            gemm(hs, blk["qkv_w"], RQ, 3 * D, D, epilogue(EPI_BF16, bias=blk["qkv_b"], out=qkv, ld_out=3 * D), st)
            sq, sk, sv = zb(B * nh, PQ, 64), zb(B * nh, PQ, 64), zb(B * nh, 64, PQ)
            _lib.check(L.ga_heads32_split(_p(qkv), _p(blk["q_n"]), _p(blk["k_n"]), RQ, nh, K, PQ, 1e-5, _p(sq), _p(sk),
                                          _p(sv), st), "heads32")
            so = torch.empty(RQ, nh * 64, device=dev, dtype=torch.bfloat16)
            _lib.check(L.ga_attention_bf16(_p(sq), _p(sk), _p(sv), _p(so), B, nh, K, K, PQ, PQ, 32 ** -0.5, 0.0, st),
                       "srt attention")
            gemm(so, blk["proj_w"], RQ, D, nh * 64, epilogue(EPI_RESID_GATE_F32, bias=blk["proj_b"], out=xs, ld_out=D), st)
            _lib.check(L.ga_layernorm_modulate(_p(xs), _p(blk["n2w"]), _p(blk["n2b"]), None, None, 0, 1, _p(hs), RQ, D, 1e-5,
                                               st), "srt norm2")
            hid = torch.empty(RQ, blk["w1"].shape[0], device=dev, dtype=torch.bfloat16)
            gemm(hs, blk["w1"], RQ, hid.shape[1], D, epilogue(EPI_GELU_BF16, bias=blk["b1"], out=hid, ld_out=hid.shape[1]), st)
            gemm(hid, blk["w2"], RQ, D, hid.shape[1], epilogue(EPI_RESID_GATE_F32, bias=blk["b2"], out=xs, ld_out=D), st)
        if acts is not None:
            acts["srt"] = xs.clone()
        zc = self.zc
        h = torch.empty(B, K, 2 * zc, device=dev)
        mean, logvar, std, lat = (torch.empty(B, K, zc, device=dev) for _ in range(4))
        _lib.check(L.ga_vae_enc_head(C.byref(self.head), _p(xs), _p(noise), RQ, D, self.head_hid, zc, _p(h), _p(mean),
                                     _p(logvar), _p(std), _p(lat), st), "readout head")
        return {"h": h, "query_pcd_xyz": qxyz, "fps_idx": qidx, "mean": mean, "logvar": logvar, "std": std,
                "latent_normalized": lat}

    def encode(self, img_to_encoder, pcd, start_idx=None, noise=None, generator=None):
        """img_to_encoder [B*V, 15, H, W] (V inner; channels rgb, normal, Pluecker ray, xyz), pcd [B, N, 3] (CUDA, fp32).
        start_idx [B]: first FPS point (default: uniform random, as random_start_point=True).  noise [B, K, zc]: the
        posterior's epsilon (default zeros: latent_normalized = mean).  Returns h [B, K, 2 zc], query_pcd_xyz and, from
        the same launch sequence, the posterior's mean / logvar / std / latent_normalized.

        The launches are captured once per (B, V, H, W, N) into a CUDA graph and replayed from static inputs;
        `use_graph = False` (or GA_B200_VAE_ENC_GRAPH=0) keeps the eager launch sequence."""
        dev = self.device
        if not img_to_encoder.is_cuda or not pcd.is_cuda:
            raise RuntimeError("gaussiananything_b200 VAE encoder needs CUDA tensors (no CPU fallback)")
        n, cin, H, W = img_to_encoder.shape
        assert cin == self.cin and n % self.V == 0, (img_to_encoder.shape, self.V)
        B = n // self.V
        assert pcd.shape[0] == B and pcd.shape[2] == 3 and pcd.shape[1] >= self.K
        if start_idx is None:
            start_idx = torch.randint(pcd.shape[1], (B,), generator=generator)
        start_idx = torch.as_tensor(start_idx).to(device=dev, dtype=torch.int32).reshape(B)
        if noise is None:
            noise = torch.zeros(B, self.K, self.zc, device=dev)
        img = img_to_encoder.float().contiguous()
        pc = pcd.float().contiguous()
        noise = noise.to(dev).float().contiguous()
        with torch.cuda.device(dev):
            return self._graphs.run((B, self.V, H, W, pc.shape[1]), self._launches, (img, pc, start_idx, noise))

    def vae_reparameterization(self, latent, sample_posterior=True, generator=None):
        """latent: encode()'s dict.  Returns latent_normalized [B, K, zc], query_pcd_xyz and the posterior."""
        post = Posterior(latent["mean"], latent["logvar"], latent["std"])
        z = post.sample(generator) if sample_posterior else post.mode()
        return {"latent_normalized": z, "posterior": post, "query_pcd_xyz": latent["query_pcd_xyz"]}


def random_state_dict(ch=64, ch_mult=(1, 2, 4, 4), in_channels=15, z_channels=10, seed=0, device="cpu"):
    """A state_dict with the reference AE's encoder keys (plus the decoder's quant_conv) and random weights: norms
    near 1 / 0, weights ~ N(0, 1/fan_in); for tests and benchmarks (there is no network for checkpoints)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shp in _expected_keys(ch=ch, ch_mult=tuple(ch_mult), in_channels=in_channels, z_channels=z_channels).items():
        leaf = k.rsplit(".", 1)[1]
        is_norm = any(s in k for s in ("norm", "q_norm", "k_norm")) and len(shp) == 1
        if is_norm and leaf == "weight":
            sd[k] = 1.0 + 0.1 * torch.randn(shp, generator=g)
        elif leaf == "bias":
            sd[k] = 0.05 * torch.randn(shp, generator=g)
        else:
            fan_in = 1
            for s in shp[1:]:
                fan_in *= s
            sd[k] = torch.randn(shp, generator=g) / fan_in ** 0.5
    return {k: v.to(device) for k, v in sd.items()}


def encode_flops(B=1, V=8, H=512, W=512, ch=64, ch_mult=(1, 2, 4, 4), in_channels=15, K=768, z_channels=10):
    """Multiply-add x 2 count of one encode (convs, the 1x1 GEMMs, mid.attn_1, the readout)."""
    f = 0
    n = B * V
    c = ch
    f += 2 * n * H * W * 9 * in_channels * ch
    cin = ch
    for i, m in enumerate(ch_mult):
        co = ch * m
        f += 2 * n * H * W * 9 * (cin * co + co * co) + (2 * n * H * W * cin * co if cin != co else 0)
        cin = co
        if i != len(ch_mult) - 1:
            H, W = (H - 2) // 2 + 1, (W - 2) // 2 + 1
            f += 2 * n * H * W * 9 * co * co
    D, inner = cin, 512
    HW = H * W
    R = n * HW
    f += 2 * 2 * R * 9 * 2 * D * D                        # mid.block_1 / block_2
    f += 2 * R * D * inner * 2                             # proj_in / proj_out
    f += 2 * R * inner * inner * 4 * 2                     # attn1 / attn2 qkv + out
    f += 4 * B * (V * HW) ** 2 * inner + 4 * n * HW ** 2 * inner
    f += 2 * R * inner * 8 * inner + 2 * R * 4 * inner * inner
    f += 2 * R * 64 * D + 2 * R * D * 2 * inner + 2 * B * K * D * inner * 2 + 4 * B * K * V * HW * inner
    f += 3 * (2 * B * K * D * 4 * D + 4 * B * K * K * D + 2 * B * K * D * 8 * D)
    return f
