"""VAE decode path latent tokens -> surfels (SURVEY.md section 8f row N1) on the library's kernels.

Mirrors what the reference's deployed decoder class does between DiT sampling and rendering:
  vit.vit_triplane.pcd_structured_latent_space_vae_decoder_cascaded
    .vit_decode_backbone      /root/reference/vit/vit_triplane.py:1415-1427   post_quant_conv -> DiT2 (dit/dit_decoder.py)
    .vit_decode_postprocess   /root/reference/vit/vit_triplane.py:1467-1501,1645-1676   conv_sr, three cascaded up-samplers
    .forward_gaussians        /root/reference/vit/vit_triplane.py:1513-1544
`SurfelDecoder(state_dict, ...)` takes the reference module's state_dict (keys vit_decoder.*, superresolution.*);
`decode(latent_normalized, query_pcd_xyz)` returns the same entries the reference's ret_dict carries
(gaussians_base, gaussians_upsampled{,_2,_3}, gaussians).  No torch arithmetic: every op is a kernel of libga_b200.so
(wgmma GEMMs with fused epilogues, wgmma attention for the DiT2 blocks, one-warp-per-sequence attention for the
up-samplers' micro-sequences, row kernels).  bf16 tensor-core operands, fp32 residual streams.  No CPU fallback.
"""
import torch

from . import _launch, _lib
from ._launch import epilogue, gemm, ptr as _p, round_up as _round_up
from ._lib import EPI_BF16, EPI_F32, EPI_GELU_BF16, EPI_HEADS, EPI_RESID_GATE_F32


class SurfelDecoder:
    CASCADE = (("ada_CA_f4_1", 8), ("ada_CA_f4_2", 4), ("ada_CA_f4_3", 3))
    use_graph = _launch.graph_switch()

    def __init__(self, state_dict, num_heads, depth, scene_max=0.45, skip_weight=0.1, device="cuda:0"):
        self.L = _lib.lib()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("gaussiananything_b200 needs a CUDA device (no CPU fallback)")
        self.H, self.depth = int(num_heads), int(depth)
        self.scene_max, self.skip = float(scene_max), float(skip_weight)
        self.scale_factor = float(self.scene_max * 0.01 / torch.nn.functional.softplus(torch.tensor(0.0)))
        dev = self.device
        sd = state_dict
        f32 = lambda k: sd[k].detach().to(device=dev, dtype=torch.float32).contiguous()
        b16 = lambda k: sd[k].detach().to(device=dev, dtype=torch.bfloat16).contiguous()
        q = "superresolution."
        self.D = D = sd["vit_decoder.pos_embed"].shape[-1]
        assert D % 64 == 0 and D // self.H == 64, "head_dim must be 64"
        self.N = sd["vit_decoder.pos_embed"].shape[1]
        w = {}
        # post_quant_conv (timm Mlp, tanh-GELU): fc1 through the small-K embed kernel, fc2 as a GEMM with K padded to 16
        zc = sd[q + "post_quant_conv.fc1.weight"].shape[1]
        hid = sd[q + "post_quant_conv.fc1.weight"].shape[0]
        self.zc, self.pq_k = zc, _round_up(hid, 16)
        w1 = torch.zeros(self.pq_k, zc, device=dev)
        b1 = torch.zeros(self.pq_k, device=dev)
        w1[:hid], b1[:hid] = f32(q + "post_quant_conv.fc1.weight"), f32(q + "post_quant_conv.fc1.bias")
        w2 = torch.zeros(D, self.pq_k, device=dev)
        w2[:, :hid] = f32(q + "post_quant_conv.fc2.weight")
        w["pq_w1"], w["pq_b1"] = w1.contiguous(), b1
        w["pq_w2"], w["pq_b2"] = w2.to(torch.bfloat16).contiguous(), f32(q + "post_quant_conv.fc2.bias")
        w["pos"] = f32("vit_decoder.pos_embed")[0].contiguous()                      # [N, D]
        # the per-token adaLN tables of all blocks come out of one GEMM: weights stacked [depth*6D, D]
        w["ada_w"] = torch.cat([b16("vit_decoder.blocks.%d.adaLN_modulation.1.weight" % l) for l in range(self.depth)], 0).contiguous()
        w["ada_b"] = torch.cat([f32("vit_decoder.blocks.%d.adaLN_modulation.1.bias" % l) for l in range(self.depth)], 0).contiguous()
        self.blocks = [self._attn_mlp("vit_decoder.blocks.%d.attn." % l, "vit_decoder.blocks.%d.mlp." % l, f32, b16)
                       for l in range(self.depth)]
        w["sr_w"], w["sr_b"] = f32(q + "conv_sr.gaussian_pred.1.weight"), f32(q + "conv_sr.gaussian_pred.1.bias")
        self.stages = []
        for name, f in self.CASCADE:
            p = q + name + "."
            nl = 1 + max(int(k[len(p + "transformer.layers."):].split(".")[0]) for k in sd if k.startswith(p + "transformer.layers."))
            layers = []
            for l in range(nl):
                t = "%stransformer.layers.%d." % (p, l)
                blk = self._attn_mlp(t + "0.fn.", t + "1.fn.", f32, b16)
                blk.update(n1_w=f32(t + "0.norm.weight"), n1_b=f32(t + "0.norm.bias"),
                           n2_w=f32(t + "1.norm.weight"), n2_b=f32(t + "1.norm.bias"))
                layers.append(blk)
            self.stages.append(dict(f=f, layers=layers, queries=f32(p + "latent_embedding")[0].contiguous(),
                                    hn_w=f32(p + "gaussian_residual_pred.norm.weight"),
                                    hn_b=f32(p + "gaussian_residual_pred.norm.bias"),
                                    h_w=f32(p + "gaussian_residual_pred.fn.weight"),
                                    h_b=f32(p + "gaussian_residual_pred.fn.bias")))
        self.w = w
        # batch size -> graph; each graph owns its activations (GBs at the deployed size)
        self._graphs = _launch.GraphCache("GA_B200_VAE_GRAPH")

    @staticmethod
    def _attn_mlp(pa, pm, f32, b16):
        qn, kn = f32(pa + "q_norm.weight"), f32(pa + "k_norm.weight")
        return dict(qkv_w=b16(pa + "qkv.weight"), qkv_b=f32(pa + "qkv.bias"), q_n=qn, k_n=kn,
                    proj_w=b16(pa + "proj.weight"), proj_b=f32(pa + "proj.bias"),
                    w1=b16(pm + "mlp.0.weight"), b1=f32(pm + "mlp.1.bias"), w2=b16(pm + "mlp.2.weight"), b2=f32(pm + "mlp.3.bias"),
                    bound=8.16 * float(qn.abs().max()) * float(kn.abs().max()))

    def decode(self, latent_normalized, query_pcd_xyz):
        """latent_normalized [B, N, Cz], query_pcd_xyz [B, N, 3] (CUDA).  Returns the reference's ret_dict entries.

        The ~300 launches of one decode are captured once per batch size into a CUDA graph and replayed from static input
        buffers (at batch 1 the eager launch sequence is host-bound); the returned tensors are copies, so they stay
        valid across later calls.  `self.use_graph = False` (or GA_B200_VAE_GRAPH=0) keeps the eager launch sequence."""
        dev = self.device
        if not latent_normalized.is_cuda:
            raise RuntimeError("gaussiananything_b200 VAE decoder needs CUDA tensors (no CPU fallback)")
        B, N, zc = latent_normalized.shape
        assert N == self.N and zc == self.zc and query_pcd_xyz.shape == (B, N, 3)
        with torch.cuda.device(dev):               # launches go to the decoder's device, not the process's current one
            lat = latent_normalized.to(device=dev, dtype=torch.float32).contiguous()
            xyz = query_pcd_xyz.to(device=dev, dtype=torch.float32).contiguous()
            return self._aliases(self._graphs.run(B, self._decode_launches, (lat, xyz)))

    @staticmethod
    def _aliases(out):
        out["gaussians"] = out["gaussians_upsampled"]                  # forward_gaussians: "only adopt SR"
        out["pos"] = out["gaussians"][..., :3]
        out["gaussians_base_opa"] = out["gaussians_base"][..., 3:4]
        return out

    def _decode_launches(self, latent_normalized, query_pcd_xyz):
        """The launch sequence of one decode on the current stream (eager, or under graph capture)."""
        L, w, dev = self.L, self.w, self.device
        B, N, zc = latent_normalized.shape
        D, H, R, dep = self.D, self.H, B * N, self.depth
        st = _launch.stream(dev)
        z = lambda *s, dt=torch.float32: torch.empty(*s, device=dev, dtype=dt)
        bf = torch.bfloat16
        lat = latent_normalized.reshape(R, zc)
        xyz = query_pcd_xyz.reshape(R, 3)
        # ---- post_quant_conv
        h0 = z(R, self.pq_k, dt=bf)
        _lib.check(L.ga_embed_fc1(_p(lat), zc, None, 0, _p(w["pq_w1"]), _p(w["pq_b1"]), _p(h0), R, self.pq_k, st), "post_quant fc1")
        c = z(R, D)
        gemm(h0, w["pq_w2"], R, D, self.pq_k, epilogue(EPI_F32, bias=w["pq_b2"], out=c, ld_out=D), st)
        # ---- DiT2: per-token adaLN tables of every block in one GEMM on silu(c)
        cs = z(R, D, dt=bf)
        _lib.check(L.ga_silu_to_bf16(_p(c), _p(cs), R * D, st), "silu")
        MW = dep * 6 * D
        mod = z(R, MW)
        gemm(cs, w["ada_w"], R, MW, D, epilogue(EPI_F32, bias=w["ada_b"], out=mod, ld_out=MW), st)
        x = w["pos"].repeat(B, 1).contiguous()                                           # [R, D] residual stream
        Np = _round_up(N, 128)
        h, ao, hid = z(R, D, dt=bf), z(R, D, dt=bf), z(R, 4 * D, dt=bf)
        qb = torch.zeros(B * H, Np, 64, device=dev, dtype=bf)
        kb = torch.zeros(B * H, Np, 64, device=dev, dtype=bf)
        vtb = torch.zeros(B * H, 64, Np, device=dev, dtype=bf)
        for l, wb in enumerate(self.blocks):
            ch = lambda j: mod[:, (l * 6 + j) * D:(l * 6 + j + 1) * D]
            _lib.check(L.ga_layernorm_modulate(_p(x), None, None, _p(ch(0)), _p(ch(1)), MW, 1, _p(h), R, D, 1e-6, st), "norm1")
            gemm(h, wb["qkv_w"], R, 3 * D, D,
                 epilogue(EPI_HEADS, bias=wb["qkv_b"], q=qb, k=kb, vt=vtb, qn_w=wb["q_n"], kn_w=wb["k_n"], heads=H,
                          first_part=0, tok_pitch=Np, rows_per_batch=N), st)
            _lib.check(L.ga_attention_bf16(_p(qb), _p(kb), _p(vtb), _p(ao), B, H, N, N, Np, Np, 0.125, wb["bound"], st), "attention")
            gemm(ao, wb["proj_w"], R, D, D,
                 epilogue(EPI_RESID_GATE_F32, bias=wb["proj_b"], out=x, ld_out=D, gate=ch(2), gate_ld=MW,
                          rows_per_batch=1), st)
            _lib.check(L.ga_layernorm_modulate(_p(x), None, None, _p(ch(3)), _p(ch(4)), MW, 1, _p(h), R, D, 1e-6, st), "norm2")
            gemm(h, wb["w1"], R, 4 * D, D, epilogue(EPI_GELU_BF16, bias=wb["b1"], out=hid, ld_out=4 * D), st)
            gemm(hid, wb["w2"], R, D, 4 * D,
                 epilogue(EPI_RESID_GATE_F32, bias=wb["b2"], out=x, ld_out=D, gate=ch(5), gate_ld=MW,
                          rows_per_batch=1), st)
        # ---- base surfels
        base_pre = z(R, 13)
        _lib.check(L.ga_thin_linear(_p(x), None, None, 1, _p(w["sr_w"]), _p(w["sr_b"]), _p(base_pre), R, D, 13, 0.0, st), "conv_sr")
        base = z(R, 13)
        _lib.check(L.ga_surfel_cascade_pack(_p(base_pre), 0, None, _p(xyz), 3, 1, self.scene_max * 0.5 * self.skip,
                                            self.scale_factor, _p(base), None, R, st), "base pack")
        out = {"latent_from_vit": x.view(B, N, D), "gaussian_base_pre_activate": base_pre.view(B, N, 13),
               "gaussians_base": base.view(B, N, 13)}
        # ---- cascaded up-samplers
        parents, prev_f, parent_g, parent_pre, S = x, 0, base, base_pre, R
        for si, stg in enumerate(self.stages):
            f = stg["f"]
            Lq = 1 + f
            Ms = S * Lq
            seq = z(Ms, D)
            _lib.check(L.ga_micro_seq_build(_p(parents), prev_f, _p(stg["queries"]), _p(seq), S, f, D, st), "seq build")
            hs, qkv, aos, hids = z(Ms, D, dt=bf), z(Ms, 3 * D, dt=bf), z(Ms, D, dt=bf), z(Ms, 4 * D, dt=bf)
            for lw in stg["layers"]:
                _lib.check(L.ga_layernorm_modulate(_p(seq), _p(lw["n1_w"]), _p(lw["n1_b"]), None, None, 0, 1, _p(hs), Ms, D, 1e-5, st), "sr norm1")
                gemm(hs, lw["qkv_w"], Ms, 3 * D, D, epilogue(EPI_BF16, bias=lw["qkv_b"], out=qkv, ld_out=3 * D), st)
                _lib.check(L.ga_micro_attention_bf16(_p(qkv), _p(lw["q_n"]), _p(lw["k_n"]), _p(aos), S, Lq, H, 1e-5, st), "micro attention")
                gemm(aos, lw["proj_w"], Ms, D, D,
                     epilogue(EPI_RESID_GATE_F32, bias=lw["proj_b"], out=seq, ld_out=D, rows_per_batch=1), st)
                _lib.check(L.ga_layernorm_modulate(_p(seq), _p(lw["n2_w"]), _p(lw["n2_b"]), None, None, 0, 1, _p(hs), Ms, D, 1e-5, st), "sr norm2")
                gemm(hs, lw["w1"], Ms, 4 * D, D, epilogue(EPI_GELU_BF16, bias=lw["b1"], out=hids, ld_out=4 * D), st)
                gemm(hids, lw["w2"], Ms, D, 4 * D,
                     epilogue(EPI_RESID_GATE_F32, bias=lw["b2"], out=seq, ld_out=D, rows_per_batch=1), st)
            res = z(Ms, 13)
            _lib.check(L.ga_thin_linear(_p(seq), _p(stg["hn_w"]), _p(stg["hn_b"]), 0, _p(stg["h_w"]), _p(stg["h_b"]), _p(res), Ms, D, 13,
                                        1e-5, st), "residual head")
            Rc = S * f
            g, pre = z(Rc, 13), z(Rc, 13)
            _lib.check(L.ga_surfel_cascade_pack(_p(res), 1, _p(parent_pre), _p(parent_g), 13, f, self.scene_max * 0.5,
                                                self.scale_factor, _p(g), _p(pre), Rc, st), "cascade pack")
            out["gaussians_upsampled" + ("" if si == 0 else "_%d" % (si + 1))] = g.view(B, Rc // B, 13)
            parents, prev_f, parent_g, parent_pre, S = seq, f, g, pre, Rc
        return out


def random_state_dict(D=768, depth=12, zc=10, seed=0, device="cpu"):
    """A state_dict with the reference decoder's key layout and shapes (vit_triplane.py:1316-1345,1614-1640) and
    random weights -- for benchmarks and size tests (there is no network for checkpoints)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}

    def lin(name, n_out, n_in, bias=True):
        sd[name + ".weight"] = torch.randn(n_out, n_in, generator=g) / n_in ** 0.5
        if bias:
            sd[name + ".bias"] = torch.randn(n_out, generator=g) * 0.02

    def attn_mlp(pa, pm):
        lin(pa + "qkv", 3 * D, D)
        lin(pa + "proj", D, D)
        sd[pa + "q_norm.weight"] = 1.0 + 0.1 * torch.randn(64, generator=g)
        sd[pa + "k_norm.weight"] = 1.0 + 0.1 * torch.randn(64, generator=g)
        sd[pm + "mlp.0.weight"] = torch.randn(4 * D, D, generator=g) / D ** 0.5
        sd[pm + "mlp.1.bias"] = torch.randn(4 * D, generator=g) * 0.02
        sd[pm + "mlp.2.weight"] = torch.randn(D, 4 * D, generator=g) / (4 * D) ** 0.5
        sd[pm + "mlp.3.bias"] = torch.randn(D, generator=g) * 0.02

    sd["vit_decoder.pos_embed"] = torch.randn(1, D, D, generator=g) * 0.02          # token count == width (reference)
    for l in range(depth):
        p = "vit_decoder.blocks.%d." % l
        attn_mlp(p + "attn.", p + "mlp.")
        sd[p + "adaLN_modulation.1.weight"] = torch.randn(6 * D, D, generator=g) * 0.02
        sd[p + "adaLN_modulation.1.bias"] = torch.randn(6 * D, generator=g) * 0.02
    q = "superresolution."
    lin(q + "post_quant_conv.fc1", zc, zc)
    lin(q + "post_quant_conv.fc2", D, zc)
    sd[q + "conv_sr.gaussian_pred.1.weight"] = torch.randn(13, D, generator=g) * 0.02
    sd[q + "conv_sr.gaussian_pred.1.bias"] = torch.randn(13, generator=g) * 0.1
    for (name, f), nl in zip(SurfelDecoder.CASCADE, (depth // 6 if depth == 12 else 2, 1, 1)):
        p = q + name + "."
        sd[p + "latent_embedding"] = torch.randn(1, f, D, generator=g)
        sd[p + "gaussian_residual_pred.norm.weight"] = torch.ones(D)
        sd[p + "gaussian_residual_pred.norm.bias"] = torch.zeros(D)
        sd[p + "gaussian_residual_pred.fn.weight"] = torch.randn(13, D, generator=g) * 0.02
        sd[p + "gaussian_residual_pred.fn.bias"] = torch.randn(13, generator=g) * 0.02
        for l in range(nl):
            t = "%stransformer.layers.%d." % (p, l)
            attn_mlp(t + "0.fn.", t + "1.fn.")
            for n in ("0.norm.", "1.norm."):
                sd[t + n + "weight"] = 1.0 + 0.1 * torch.randn(D, generator=g)
                sd[t + n + "bias"] = torch.randn(D, generator=g) * 0.02
    return {k: v.to(device) for k, v in sd.items()}


def decode_flops(D=768, depth=12, N=None):
    """Multiply-add x 2 count of one sample (tools/n1_cost.py): DiT2 blocks + the per-token adaLN GEMM + three
    up-sampler stages of depth (2 if depth != 12 else depth // 6), 1, 1."""
    N = D if N is None else N
    blk = lambda Ls: 2 * Ls * D * (3 * D + D + 8 * D) + 4 * Ls * Ls * D
    d1 = depth // 6 if depth == 12 else 2
    return (depth * (blk(N) + 2 * N * D * 6 * D) + N * d1 * blk(9) + N * 8 * blk(5) + N * 32 * blk(4))


# ---------------------------------------------------------------------------------------------------------------
# Drop-in for the reference's auto-encoder wrapper on the decode / render behaviours (SURVEY.md 8f rows N1, N2)
# ---------------------------------------------------------------------------------------------------------------
class SurfelAE:
    """Mirror of `nsr.script_util.AE.forward` (/root/reference/nsr/script_util.py:300-367) for the behaviours the
    sampling pipeline uses after the DiT (/root/reference/nsr/lsgm/flow_matching_trainer.py:1399-1424,1545-1567):

      rec_model(latent={'latent_normalized': [B,N,Cz], 'query_pcd_xyz': [B,N,3]}, behaviour='decode_gs_after_vae_no_render')
      rec_model(img=None, c=c, latent=ret, behaviour='triplane_dec', bg_color=..., render_all_scale=True)
      rec_model(latent=..., c=c, behaviour='decode_after_vae')

    `triplane_decode` (/root/reference/vit/vit_triplane.py:1550-1591) renders every level of detail of the cascade --
    gaussians_base 128^2, gaussians_upsampled 256^2, _2 384^2, _3 512^2 -- for all B x V cameras.  The reference
    issues 4 x B x V sequential launch sets from Python; here every level is ONE batched launch set and the four
    levels run on four CUDA streams, so the small levels (768 / 6 144 / 24 576 surfels: latency bound) overlap with
    the 73 728-surfel one.  With `encoder=` (vae_encoder.SurfelEncoder) the encoder behaviours 'enc', 'encoder_vae' and
    'enc_dec_wo_triplane' run too; without one, and for the other training behaviours, they raise."""

    OUTPUT_SIZE = {"gaussians_base": 128, "gaussians_upsampled": 256, "gaussians_upsampled_2": 384,
                   "gaussians_upsampled_3": 512}

    def __init__(self, decoder, renderer=None, img_size=None, rand_base_render=True, rendering_kwargs=None, encoder=None):
        from .gs_surfel import GaussianRenderer2DGS
        self.decoder = decoder
        self.encoder = encoder          # vae_encoder.SurfelEncoder: enables 'enc', 'encoder_vae', 'enc_dec_wo_triplane'
        self.img_size = img_size
        self.output_size = dict(self.OUTPUT_SIZE)
        self.rand_base_render = rand_base_render
        self.rendering_kwargs = rendering_kwargs or {}
        self.gs = renderer if renderer is not None else GaussianRenderer2DGS(512, 3, self.rendering_kwargs)
        self._streams = None

    # ---- reference method names
    def decode_after_vae_no_render(self, ret_dict, img_size=None):
        lat = ret_dict["latent_normalized"] if isinstance(ret_dict, dict) else ret_dict
        out = dict(ret_dict) if isinstance(ret_dict, dict) else {}
        out.update(self.decoder.decode(lat, ret_dict["query_pcd_xyz"]))
        return out

    def decode_after_vae_no_render_gs(self, ret_dict, img_size=None):
        return self.decode_after_vae_no_render(ret_dict, img_size)          # decode() already applies forward_gaussians

    def decode_after_vae(self, ret_dict, c, img_size=None, return_raw_only=False):
        return self.triplane_decode(self.decode_after_vae_no_render(ret_dict, img_size), c)

    def triplane_decode(self, ret_after_gaussian_forward, c, bg_color=None, render_all_scale=False, **kwargs):
        import random
        keys = list(self.output_size.keys())
        if self.rand_base_render and not render_all_scale:
            keys = [random.choice(keys[:-1])] + [keys[-1]]
        dev = ret_after_gaussian_forward[keys[-1]].device
        main = torch.cuda.current_stream(dev)
        if self._streams is None or self._streams[0].device != dev:
            self._streams = [torch.cuda.Stream(dev) for _ in range(len(self.output_size))]
        tanfov = c["tanfov"]
        tanfov = float(tanfov) if not isinstance(tanfov, float) else tanfov
        fork = torch.cuda.Event()
        fork.record(main)
        results = {}
        # largest level first: it is the long pole, the small ones fill in beside it
        for i, key in enumerate(sorted(keys, key=lambda k: -self.output_size[k])):
            s = self._streams[i]
            s.wait_event(fork)
            with torch.cuda.stream(s):
                r = self.gs.render(ret_after_gaussian_forward[key], c["cam_view"], c["cam_view_proj"], c["cam_pos"],
                                   tanfov=tanfov, bg_color=bg_color, output_size=self.output_size[key])
                r["image_raw"] = r["image"] * 2 - 1                      # [0,1] -> [-1,1] (vit_triplane.py:1570-1573)
                r["image_depth"] = r["depth"]
                r["image_mask"] = r["alpha"]
                for t in r.values():
                    t.record_stream(main)
            results[key] = r
        for s in self._streams:
            main.wait_stream(s)
        return {k: results[k] for k in keys}                              # the reference's key order

    def forward(self, img=None, c=None, latent=None, behaviour="enc_dec", coordinates=None, directions=None,
                return_raw_only=False, *args, **kwargs):
        if behaviour == "decode_gs_after_vae_no_render":
            return self.decode_after_vae_no_render_gs(latent, self.img_size)
        if behaviour == "decode_after_vae_no_render":
            return self.decode_after_vae_no_render(latent, self.img_size)
        if behaviour == "decode_after_vae":
            return self.decode_after_vae(latent, c, self.img_size)
        if behaviour == "triplane_dec":
            assert latent is not None
            return self.triplane_decode(latent, c, **kwargs)
        if behaviour == "get_rendering_kwargs":
            return self.rendering_kwargs
        if self.encoder is not None and behaviour in ("enc", "encoder_vae", "enc_dec_wo_triplane"):
            return self._encoder_behaviour(behaviour, img, kwargs)
        raise NotImplementedError("gaussiananything_b200.SurfelAE: behaviour %r is outside the decode / render path "
                                  "(encoder and training behaviours are not rebuilt: SURVEY.md section 8)" % (behaviour,))

    __call__ = forward

    def _encoder_behaviour(self, behaviour, img, kwargs):
        """nsr/script_util.py:320-359 with the point-cloud-structured encoder: img = img_to_encoder [B*V, 15, H, W],
        pcd= [B, N, 3]; optional fps_start= [B] and generator= (posterior noise, FPS start)."""
        enc = self.encoder
        pcd, gen = kwargs.get("pcd"), kwargs.get("generator")
        if pcd is None:
            raise ValueError("SurfelAE(behaviour=%r) needs pcd= [B, N, 3]" % (behaviour,))
        B = img.shape[0] // enc.V
        if behaviour == "enc":
            return enc.encode(img, pcd, kwargs.get("fps_start"), generator=gen)
        if behaviour == "encoder_vae":
            return enc.vae_reparameterization(enc.encode(img, pcd, kwargs.get("fps_start"), generator=gen), True, gen)
        # enc_dec_wo_triplane: the posterior is sampled inside the encoder's launch sequence (mean + std * eps)
        eps = torch.randn(B, enc.K, enc.zc, generator=gen)
        lat = enc.encode(img, pcd, kwargs.get("fps_start"), noise=eps.to(img.device), generator=gen)
        from .vae_encoder import Posterior
        ret = {"latent_normalized": lat["latent_normalized"], "query_pcd_xyz": lat["query_pcd_xyz"],
               "posterior": Posterior(lat["mean"], lat["logvar"], lat["std"]), "h": lat["h"]}
        return self.decode_after_vae_no_render(ret, self.img_size)
