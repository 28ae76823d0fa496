"""Mirror of the deployed image-to-3D DiT denoisers of the reference:

  dit.dit_i23d.DiT_I23D_PCD_PixelArt_noclip               (/root/reference/dit/dit_i23d.py:437-567)
  dit.dit_i23d.DiT_I23D_PCD_PixelArt_noclip_clay_stage2   (/root/reference/dit/dit_i23d.py:664-750)
  block ImageCondDiTBlockPixelArtRMSNormClayLRM           (/root/reference/dit/dit_models_xformers.py:717-787)
  registry DiT_models                                     (/root/reference/dit/dit_i23d.py:1665-1697)

Same constructor arguments, attribute names and state_dict key layout (a
reference checkpoint loads with strict=True), same `forward(x, timesteps,
context)` / `forward_with_cfg(x, t, context, cfg_scale)` contracts.  The
forward pass does no arithmetic in torch: every op is a kernel of
libga_b200.so (wgmma GEMMs with fused epilogues, wgmma flash attention,
fused RMSNorm+modulate, ...) enqueued on the current CUDA stream, optionally
replayed from a CUDA graph.  There is no CPU / eager fallback.

Precision: GEMM / attention operands bf16 (the reference runs them under bf16
autocast), fp32 accumulation, fp32 residual stream, fp32 norms, fp32 output.
"""
import math

import torch
import torch.nn as nn

from . import _launch, _lib, dit_grad
from ._launch import epilogue, gemm, ptr as _p, round_up as _round_up
from ._lib import EPI_F32, EPI_GELU_BF16, EPI_HEADS, EPI_RESID_GATE_F32
# dit.EPI_*, dit.GaGemmEpilogue, dit._gemm_config and dit._p: earlier homes of these names, still read by tools and tests
from ._launch import gemm_config as _gemm_config  # noqa: F401
from ._lib import EPI_BF16, GaGemmEpilogue  # noqa: F401

_bind = _lib.lib


# --------------------------------------------------------------------------
# parameter containers with the reference's names (no forward of their own)
# --------------------------------------------------------------------------
class _Weight(nn.Module):
    def __init__(self, n, init=1.0):
        super().__init__()
        self.weight = nn.Parameter(torch.full((n,), float(init)))


class _Bias(nn.Module):
    def __init__(self, n):
        super().__init__()
        self.bias = nn.Parameter(torch.zeros(n))


class _Mlp(nn.Module):          # timm Mlp layout: fc1, fc2
    def __init__(self, cin, hidden, cout):
        super().__init__()
        self.fc1 = nn.Linear(cin, hidden)
        self.fc2 = nn.Linear(hidden, cout)


class _SelfAttn(nn.Module):
    def __init__(self, dim, heads):
        super().__init__()
        self.qkv = nn.Linear(dim, 3 * dim, bias=True)
        self.proj = nn.Linear(dim, dim)
        self.q_norm = _Weight(dim // heads)
        self.k_norm = _Weight(dim // heads)


class _CrossAttn(nn.Module):
    def __init__(self, dim, ctx_dim, heads):
        super().__init__()
        self.to_q = nn.Linear(dim, dim, bias=False)
        self.to_k = nn.Linear(ctx_dim, dim, bias=False)
        self.q_norm = _Weight(dim // heads)
        self.k_norm = _Weight(dim // heads)
        self.to_v = nn.Linear(ctx_dim, dim, bias=False)
        self.to_out = nn.Sequential(nn.Linear(dim, dim), nn.Dropout(0.0))


class _FusedMLP(nn.Module):     # xformers FusedMLP key layout: mlp.{0.weight, 1.bias, 2.weight, 3.bias}
    def __init__(self, dim, mult):
        super().__init__()
        self.mlp = nn.Sequential(nn.Linear(dim, mult * dim, bias=False), _Bias(mult * dim),
                                 nn.Linear(mult * dim, dim, bias=False), _Bias(dim))


class ImageCondDiTBlockPixelArtRMSNormClayLRM(nn.Module):
    """Parameter layout of /root/reference/dit/dit_models_xformers.py:717-763 (CA -> gated SA -> gated FFN), with the
    reference's forward (:765-787) as a differentiable call of dit_grad.block_forward for training."""

    def __init__(self, hidden_size, num_heads, context_dim, mlp_ratio=4, **kw):
        super().__init__()
        self.num_heads = num_heads
        self.scale_shift_table = nn.Parameter(torch.randn(6, hidden_size) / hidden_size ** 0.5)
        self.norm1 = _Weight(hidden_size)
        self.norm2 = _Weight(hidden_size)
        self.attn = _SelfAttn(hidden_size, num_heads)
        self.mlp = _FusedMLP(hidden_size, int(mlp_ratio))
        self.attention_y_norm = _Weight(1024)                    # present, unused (reference :456-458)
        self.cross_attn_dino = _CrossAttn(hidden_size, context_dim, num_heads)
        self.prenorm_ca_dino = _Weight(hidden_size)
        self.adaLN_modulation = None

    def forward(self, x, t, dino_spatial_token, clip_caption_token=None, freqs_cis=None, **kwargs):
        """x [B, N, D] + cross-attention on dino_spatial_token [B, M, Dc], gated self-attention and gated FFN
        modulated by scale_shift_table + t (t [B, 6 D]).  clip_caption_token is ignored, as in the reference, where
        the text cross-attention returns zeros; freqs_cis (RoPE) raises NotImplementedError."""
        return dit_grad.block_forward(self, x, t, dino_spatial_token, freqs_cis=freqs_cis)


class _TimestepEmbedder(nn.Module):
    def __init__(self, hidden, freq=256):
        super().__init__()
        self.mlp = nn.Sequential(nn.Linear(freq, hidden), nn.SiLU(), nn.Linear(hidden, hidden))
        self.frequency_embedding_size = freq


class _FinalLayer(nn.Module):   # T2IFinalLayer (/root/reference/dit/dit_models_xformers.py:62-85)
    def __init__(self, hidden, out_channels):
        super().__init__()
        self.linear = nn.Linear(hidden, out_channels)
        self.scale_shift_table = nn.Parameter(torch.randn(2, hidden) / hidden ** 0.5)
        self.adaLN_modulation = None
        self.out_channels = out_channels


class _CaptionEmbedder(nn.Module):
    def __init__(self, cin, hidden):
        super().__init__()
        self.y_proj = _Mlp(cin, hidden, hidden)


class _XYZPosEmbed(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.xyz_projection = nn.Linear(63, dim)


class DiT_I23D_PCD_PixelArt_noclip(nn.Module):
    xyz_cond = False        # True for the stage-2 models: context["fps-xyz"] conditions the tokens

    def __init__(self, input_size=32, patch_size=2, in_channels=4, hidden_size=1152, depth=28, num_heads=16,
                 mlp_ratio=4, class_dropout_prob=0.1, num_classes=1000, learn_sigma=True, mixing_logit_init=-3,
                 mixed_prediction=True, context_dim=False, pooling_ctx_dim=768, roll_out=False, vit_blk=None,
                 final_layer_blk=None, create_cap_embedder=True, use_clay_ca=False, has_caption=False,
                 rope_scaling_factor=1.0, ntk_factor=1.0, enable_rope=False, **kw):
        super().__init__()
        if enable_rope:
            raise NotImplementedError("enable_rope=True is dead code in the reference (SURVEY.md F6)")
        if has_caption:
            raise NotImplementedError("caption conditioning is not on the deployed i23d path")
        if hidden_size % num_heads or hidden_size // num_heads != 64:
            raise ValueError("the attention kernel is specialised for head_dim 64 (all reference archs)")
        assert roll_out
        self.depth, self.mlp_ratio, self.learn_sigma = depth, mlp_ratio, learn_sigma
        self.in_channels = in_channels
        self.out_channels = in_channels * 2 if learn_sigma else in_channels
        self.patch_size, self.num_heads, self.embed_dim = patch_size, num_heads, hidden_size
        self.roll_out, self.plane_n, self.context_dim = roll_out, 3, context_dim
        self.enable_rope, self.freqs_cis, self.use_clay_ca, self.has_caption = False, None, use_clay_ca, False
        self.x_embed_in = in_channels
        self.x_embedder = _Mlp(in_channels, hidden_size, hidden_size)
        self.t_embedder = _TimestepEmbedder(hidden_size)
        self.y_embedder = None
        self.blocks = nn.ModuleList([
            ImageCondDiTBlockPixelArtRMSNormClayLRM(hidden_size, num_heads, context_dim, mlp_ratio)
            for _ in range(depth)])
        self.final_layer = _FinalLayer(hidden_size, self.out_channels)
        self.clip_spatial_proj = _CaptionEmbedder(1024, hidden_size)          # present, unused
        self.adaLN_modulation = nn.Sequential(nn.SiLU(), nn.Linear(hidden_size, 6 * hidden_size))
        self.cap_embedder = nn.Sequential(nn.LayerNorm(pooling_ctx_dim), nn.Linear(pooling_ctx_dim, hidden_size)) \
            if create_cap_embedder else nn.Identity()
        self.attention_y_norm = _Weight(1024)                                  # present, unused
        self.pooled_vec_embedder = nn.Sequential(nn.LayerNorm(context_dim), nn.Linear(context_dim, hidden_size))
        self.initialize_weights()
        self._engine = None
        self.cfg_dedup = False             # opt-in: skip the duplicate CFG half when uc == c bit for bit (forward_with_cfg)

    # reference init (dit_models_xformers.py:1117-1159, dit_i23d.py:213-214,508-509)
    def initialize_weights(self):
        for m in self.modules():
            if isinstance(m, nn.Linear):
                nn.init.xavier_uniform_(m.weight)
                if m.bias is not None:
                    nn.init.constant_(m.bias, 0)
        nn.init.normal_(self.t_embedder.mlp[0].weight, std=0.02)
        nn.init.normal_(self.t_embedder.mlp[2].weight, std=0.02)
        for lin in (self.final_layer.linear, self.adaLN_modulation[1], self.pooled_vec_embedder[1]):
            nn.init.constant_(lin.weight, 0)
            nn.init.constant_(lin.bias, 0)
        if isinstance(self.cap_embedder, nn.Sequential):
            nn.init.constant_(self.cap_embedder[1].weight, 0)
            nn.init.constant_(self.cap_embedder[1].bias, 0)

    def randomize_zero_init_(self, std=0.02, seed=0):
        """SURVEY.md 8(d): the zero-initialised tensors would make the output identically 0."""
        g = torch.Generator().manual_seed(seed)
        for lin in (self.final_layer.linear, self.adaLN_modulation[1], self.pooled_vec_embedder[1]):
            lin.weight.data.copy_(torch.randn(lin.weight.shape, generator=g) * std)
            lin.bias.data.copy_(torch.randn(lin.bias.shape, generator=g) * std)
        self.invalidate()
        return self

    def invalidate(self):
        """Call after changing parameters in place (the bf16 weight pack is cached)."""
        self._engine = None

    def load_state_dict(self, *a, **k):
        r = super().load_state_dict(*a, **k)
        self.invalidate()
        return r

    def _apply(self, fn, *a, **k):
        r = super()._apply(fn, *a, **k)
        self._engine = None
        return r

    # ------------------------------------------------------------------ forward
    def _extra_embed(self, context):
        return None, None          # stage 1: no xyz conditioning

    def _engine_for(self, x, context):
        assert isinstance(context, dict)
        if not x.is_cuda:
            raise RuntimeError("gaussiananything_b200 DiT needs CUDA tensors: there is no CPU fallback")
        if torch.is_grad_enabled():
            # inference-only mirror (SURVEY.md 8a: the denoiser FORWARD under the ODE sampler): nothing here records
            # an autograd graph, so a caller expecting gradients must be told instead of silently getting none
            wants = x.requires_grad or any(isinstance(v, torch.Tensor) and v.requires_grad for v in context.values())
            if wants or (self.training and any(p.requires_grad for p in self.parameters())):
                raise RuntimeError(
                    "gaussiananything_b200 DiT is inference-only (no autograd through the CUDA kernels): call it under "
                    "torch.no_grad() / torch.inference_mode(), or after .eval() with inputs that do not require grad")
        if self._engine is None or self._engine.device != x.device:
            self._engine = self._new_engine(x.device)
        elif self._engine.param_versions != _param_versions(self):
            self._engine = self._new_engine(x.device)          # parameters changed in place: stale bf16 pack / graph
        return self._engine

    def _new_engine(self, device):
        return _DiTEngine(self, device)

    def forward(self, x, timesteps=None, context=None, y=None, get_attr='', **kwargs):
        return self._engine_for(x, context).run(x, timesteps, context, cfg_scale=None)

    def forward_with_cfg(self, x, t, context, cfg_scale):
        """/root/reference/dit/dit_i23d.py:159-172: one 2B forward, u + s (c - u), duplicated.

        `self.cfg_dedup = True` (opt-in, SURVEY.md F13): when the conditional and unconditional halves of x, t and
        every context tensor are bit-identical -- the reference's stage-2 call, where `uc == c`
        (nsr/lsgm/flow_matching_trainer.py:2004, sgm/modules/encoders/modules.py:166-168) -- u + s (c - u) == c
        exactly, so only B rows are evaluated and duplicated.  Same bits as the 2B call (tests/test_dit_gpu.py)."""
        eng = self._engine_for(x, context)
        if getattr(self, "cfg_dedup", False) and x.shape[0] % 2 == 0 and eng.halves_identical(x, t, context):
            h = x.shape[0] // 2
            ctx_h = eng.half_context(context)
            y = eng.run(x[:h], t[:h] if t.numel() > 1 else t, ctx_h, cfg_scale=None)
            return torch.cat([y, y], 0)
        return eng.run(x, t, context, cfg_scale=float(cfg_scale))


def _param_versions(model):
    """Sum of the parameters' in-place version counters (an optimizer step / .data.copy_ / load bumps it)."""
    tot = 0
    for p in model.parameters():
        try:
            tot += p._version
        except RuntimeError:              # inference tensors do not track versions
            pass
    return tot


class DiT_I23D_PCD_PixelArt_noclip_clay_stage2(DiT_I23D_PCD_PixelArt_noclip):
    xyz_cond = True

    def __init__(self, *a, use_pe_cond=False, **kw):
        super().__init__(*a, **kw)
        self.has_caption = False
        self.use_pe_cond = use_pe_cond
        extra = 0 if use_pe_cond else 3
        self.x_embed_in = self.in_channels + extra
        self.x_embedder = _Mlp(self.in_channels + extra, self.embed_dim, self.embed_dim)
        nn.init.xavier_uniform_(self.x_embedder.fc1.weight); nn.init.constant_(self.x_embedder.fc1.bias, 0)
        nn.init.xavier_uniform_(self.x_embedder.fc2.weight); nn.init.constant_(self.x_embedder.fc2.bias, 0)
        if use_pe_cond:
            self.xyz_pos_embed = _XYZPosEmbed(self.embed_dim)
            nn.init.xavier_uniform_(self.xyz_pos_embed.xyz_projection.weight)
            nn.init.constant_(self.xyz_pos_embed.xyz_projection.bias, 0)


# --------------------------------------------------------------------------
# engine: bf16 weight pack + workspaces + launch sequence (+ CUDA graph)
# --------------------------------------------------------------------------
_ATTN_SCALE = 1.0 / math.sqrt(64.0)        # softmax scale of head_dim 64


class _DiTEngine:
    """The image model's engine.  The text-to-3D engine (dit_t23d._T23DEngine) overrides only the class attributes
    below, the final layer's modulation and the context K/V with its per-block context norm."""
    ctx_key, vec_key = "img_crossattn", "img_vector"          # the conditioner's output keys this model reads
    block_order = ("cross_attn", "self_attn", "ffn")          # the sublayer methods each block launches, in order
    vec_embedder = "pooled_vec_embedder"                      # the model's LayerNorm + Linear of the pooled vector
    ca_modules = ("cross_attn_dino", "prenorm_ca_dino")       # a block's cross-attention and its pre-norm

    def __init__(self, model, device):
        self.L = _bind()
        self.device = device
        self.m = model
        self.D, self.H, self.depth = model.embed_dim, model.num_heads, model.depth
        self.Cin, self.Cout = model.in_channels, model.out_channels
        self.Dc = model.context_dim
        self.stage2 = model.xyz_cond
        self.use_pe = self.stage2 and model.use_pe_cond
        self.use_graph = True
        self.tap_blocks = False            # tests: keep the residual stream after every block (s["taps"][l])
        self.param_versions = _param_versions(model)
        with torch.inference_mode(False), torch.cuda.device(device):
            self._pack()
        self._shape = None
        self._ctx_ref = None               # STRONG reference to the context tensor whose K/V are cached
        self._ctx_ver = None
        self._half_ctx = None
        self._graph = None

    # ---- weights
    def _f32(self, t):
        return t.detach().to(device=self.device, dtype=torch.float32).contiguous()

    def _b16(self, t):
        return t.detach().to(device=self.device, dtype=torch.bfloat16).contiguous()

    def _pack(self):
        m, dev, f32, b16 = self.m, self.device, self._f32, self._b16
        vec = getattr(m, self.vec_embedder)
        w = {}
        w["t0_w"], w["t0_b"] = f32(m.t_embedder.mlp[0].weight), f32(m.t_embedder.mlp[0].bias)
        w["t2_w"], w["t2_b"] = f32(m.t_embedder.mlp[2].weight), f32(m.t_embedder.mlp[2].bias)
        w["vec_ln_w"], w["vec_ln_b"] = f32(vec[0].weight), f32(vec[0].bias)
        w["vec_w"], w["vec_b"] = f32(vec[1].weight), f32(vec[1].bias)
        w["ada_w"], w["ada_b"] = f32(m.adaLN_modulation[1].weight), f32(m.adaLN_modulation[1].bias)
        w["fc1_w"], w["fc1_b"] = f32(m.x_embedder.fc1.weight), f32(m.x_embedder.fc1.bias)
        w["fc2_w"], w["fc2_b"] = b16(m.x_embedder.fc2.weight), f32(m.x_embedder.fc2.bias)
        if self.use_pe:
            wx = torch.zeros(self.D, 64, device=dev, dtype=torch.float32)
            wx[:, :63] = f32(m.xyz_pos_embed.xyz_projection.weight)
            w["xyz_w"], w["xyz_b"] = wx.to(torch.bfloat16).contiguous(), f32(m.xyz_pos_embed.xyz_projection.bias)
        w["tables"] = torch.stack([f32(b.scale_shift_table) for b in m.blocks]).contiguous()      # [L,6,D]
        w.update(self._pack_final_modulation())
        w["fin_w"], w["fin_b"] = f32(m.final_layer.linear.weight), f32(m.final_layer.linear.bias)
        self.w, self.wb = w, [self._pack_block(b) for b in m.blocks]

    def _pack_block(self, b):
        f32, b16 = self._f32, self._b16
        ca, pre = (getattr(b, n) for n in self.ca_modules)
        sa, mlp = b.attn, b.mlp.mlp
        # |q.k|/8 <= (sqrt(64) max|wq|)(sqrt(64) max|wk|)/8 for RMS-normalised q, k (+2% for bf16 rounding):
        # lets the attention kernel skip the running maximum (ga_b200.h: score_bound)
        bound = lambda a: 8.16 * float(a.q_norm.weight.detach().abs().max()) * float(a.k_norm.weight.detach().abs().max())
        return dict(
            pre_w=f32(pre.weight), n1_w=f32(b.norm1.weight), n2_w=f32(b.norm2.weight),
            caq_w=b16(ca.to_q.weight), cakv_w=b16(torch.cat([ca.to_k.weight, ca.to_v.weight], 0)),
            caq_n=f32(ca.q_norm.weight), cak_n=f32(ca.k_norm.weight),
            cao_w=b16(ca.to_out[0].weight), cao_b=f32(ca.to_out[0].bias),
            qkv_w=b16(sa.qkv.weight), qkv_b=f32(sa.qkv.bias), q_n=f32(sa.q_norm.weight), k_n=f32(sa.k_norm.weight),
            proj_w=b16(sa.proj.weight), proj_b=f32(sa.proj.bias),
            w1=b16(mlp[0].weight), b1=f32(mlp[1].bias), w2=b16(mlp[2].weight), b2=f32(mlp[3].bias),
            ca_bound=bound(ca), sa_bound=bound(sa))

    def _pack_final_modulation(self):
        return {"table_f": self._f32(self.m.final_layer.scale_shift_table)}

    # ---- workspaces for a (B, N, M) problem
    def _alloc(self, B, N, M):
        dev, D, H = self.device, self.D, self.H
        R = B * N
        z = lambda *s, dt=torch.float32: torch.zeros(*s, device=dev, dtype=dt)
        bf = torch.bfloat16
        self.Np, self.Mp = _round_up(N, 128), _round_up(M, 128)
        s = dict(
            x_in=z(B, N, self.Cin), t_in=z(B), vec_in=z(B, self.Dc), y=z(B, N, self.Cout), y_cfg=z(B, N, self.Cout),
            sinus=z(B, 256), h1=z(B, D), temb=z(B, D), vln=z(B, self.Dc), t0=z(B, 6 * D),
            mod=z(self.depth, B, 6 * D), modf=z(B, 2 * D),
            e1=z(R, D, dt=bf), xres=z(R, D), h=z(R, D, dt=bf), ao=z(R, D, dt=bf), hid=z(R, 4 * D, dt=bf),
            q=z(B * H, self.Np, 64, dt=bf), k=z(B * H, self.Np, 64, dt=bf), vt=z(B * H, 64, self.Np, dt=bf),
            ctx=z(B * M, self.Dc, dt=bf),
            kc=z(self.depth, B * H, self.Mp, 64, dt=bf), vtc=z(self.depth, B * H, 64, self.Mp, dt=bf))
        if self.stage2:
            s["xyz_in"] = z(B, N, 3)
            if self.use_pe:
                s["pe"] = z(R, 64, dt=bf)
        self.s = s
        self._shape = (B, N, M)
        self._graph = None
        self._ctx_ref = None

    # ---- launches
    _epi = staticmethod(epilogue)          # bench.py builds its isolated-GEMM epilogue through the engine

    def _context_kv(self, st, c32):
        """Timestep-independent cross-attention K/V of every block: once per context (SURVEY.md F11).
        c32: the context tokens [B*M, Dc] fp32."""
        B, N, M = self._shape
        s, D, H = self.s, self.D, self.H
        _lib.check(self.L.ga_f32_to_bf16(_p(c32), _p(s["ctx"]), c32.numel(), st), "ctx->bf16")
        for l, wb in enumerate(self.wb):
            e = epilogue(EPI_HEADS, k=s["kc"][l], vt=s["vtc"][l], kn_w=wb["cak_n"], heads=H, first_part=1,
                         tok_pitch=self.Mp, rows_per_batch=M)
            gemm(s["ctx"], wb["cakv_w"], B * M, 2 * D, self.Dc, e, st)

    def _final_modulation(self, st):
        """modf [B, 2D] = final_layer.scale_shift_table + temb (T2IFinalLayer)."""
        B, D = self._shape[0], self.D
        _lib.check(self.L.ga_add_tables(_p(self.w["table_f"]), _p(self.s["temb"]), _p(self.s["modf"]), 1, B, 2 * D, D, st),
                   "final modulation")

    # ---- the block's sublayers: launches that update the residual stream xres.  l: the block's index, wb: its
    # weights, ch: its six [B, D] modulation chunks (shift, scale and gate of the self-attention, then of the FFN)
    def cross_attn(self, st, l, wb, ch):
        """xres += CA(RMSNorm(xres; pre-norm)) against block l's cached context K/V: no modulation, no gate."""
        L, s = self.L, self.s
        B, N, M = self._shape
        D, H, R = self.D, self.H, B * N
        _lib.check(L.ga_rmsnorm_modulate(_p(s["xres"]), _p(wb["pre_w"]), None, None, 0, N, _p(s["h"]), R, D, 1e-5, st), "prenorm")
        gemm(s["h"], wb["caq_w"], R, D, D,
             epilogue(EPI_HEADS, q=s["q"], qn_w=wb["caq_n"], heads=H, first_part=0, tok_pitch=self.Np,
                      rows_per_batch=N), st)
        _lib.check(L.ga_attention_bf16(_p(s["q"]), _p(s["kc"][l]), _p(s["vtc"][l]), _p(s["ao"]), B, H, N, M, self.Np,
                                       self.Mp, _ATTN_SCALE, wb["ca_bound"], st), "cross attention")
        gemm(s["ao"], wb["cao_w"], R, D, D,
             epilogue(EPI_RESID_GATE_F32, bias=wb["cao_b"], out=s["xres"], ld_out=D, rows_per_batch=N), st)

    def self_attn(self, st, l, wb, ch):
        """xres += gate_msa * SA(RMSNorm(xres) * (1 + scale_msa) + shift_msa)."""
        L, s = self.L, self.s
        B, N, M = self._shape
        D, H, R = self.D, self.H, B * N
        _lib.check(L.ga_rmsnorm_modulate(_p(s["xres"]), _p(wb["n1_w"]), _p(ch[0]), _p(ch[1]), 6 * D, N, _p(s["h"]), R, D,
                                         1e-5, st), "norm1")
        gemm(s["h"], wb["qkv_w"], R, 3 * D, D,
             epilogue(EPI_HEADS, bias=wb["qkv_b"], q=s["q"], k=s["k"], vt=s["vt"], qn_w=wb["q_n"],
                      kn_w=wb["k_n"], heads=H, first_part=0, tok_pitch=self.Np, rows_per_batch=N), st)
        _lib.check(L.ga_attention_bf16(_p(s["q"]), _p(s["k"]), _p(s["vt"]), _p(s["ao"]), B, H, N, N, self.Np, self.Np,
                                       _ATTN_SCALE, wb["sa_bound"], st), "self attention")
        gemm(s["ao"], wb["proj_w"], R, D, D,
             epilogue(EPI_RESID_GATE_F32, bias=wb["proj_b"], out=s["xres"], ld_out=D, gate=ch[2],
                      gate_ld=6 * D, rows_per_batch=N), st)

    def ffn(self, st, l, wb, ch):
        """xres += gate_mlp * FFN(RMSNorm(xres) * (1 + scale_mlp) + shift_mlp)."""
        L, s = self.L, self.s
        B, N, M = self._shape
        D, R = self.D, B * N
        _lib.check(L.ga_rmsnorm_modulate(_p(s["xres"]), _p(wb["n2_w"]), _p(ch[3]), _p(ch[4]), 6 * D, N, _p(s["h"]), R, D,
                                         1e-5, st), "norm2")
        gemm(s["h"], wb["w1"], R, 4 * D, D, epilogue(EPI_GELU_BF16, bias=wb["b1"], out=s["hid"], ld_out=4 * D), st)
        gemm(s["hid"], wb["w2"], R, D, 4 * D,
             epilogue(EPI_RESID_GATE_F32, bias=wb["b2"], out=s["xres"], ld_out=D, gate=ch[5],
                      gate_ld=6 * D, rows_per_batch=N), st)

    def _forward_launches(self, st, cfg_scale):
        L, s, w = self.L, self.s, self.w
        B, N, M = self._shape
        D, R = self.D, B * N
        # ---- prologue: timestep + pooled vector -> adaLN tables and the final layer's modulation
        _lib.check(L.ga_timestep_sinusoid(_p(s["t_in"]), _p(s["sinus"]), B, 256, st), "sinusoid")
        _lib.check(L.ga_linear_small(_p(s["sinus"]), _p(w["t0_w"]), _p(w["t0_b"]), _p(s["h1"]), B, D, 256, 0, 1, 0, st), "t0")
        _lib.check(L.ga_linear_small(_p(s["h1"]), _p(w["t2_w"]), _p(w["t2_b"]), _p(s["temb"]), B, D, D, 0, 0, 0, st), "t2")
        _lib.check(L.ga_layernorm_rows(_p(s["vec_in"]), _p(w["vec_ln_w"]), _p(w["vec_ln_b"]), _p(s["vln"]), B, self.Dc, 1e-5, st), "ln")
        _lib.check(L.ga_linear_small(_p(s["vln"]), _p(w["vec_w"]), _p(w["vec_b"]), _p(s["temb"]), B, D, self.Dc, 0, 0, 1, st), "vec")
        _lib.check(L.ga_linear_small(_p(s["temb"]), _p(w["ada_w"]), _p(w["ada_b"]), _p(s["t0"]), B, 6 * D, D, 1, 0, 0, st), "ada")
        _lib.check(L.ga_add_tables(_p(w["tables"]), _p(s["t0"]), _p(s["mod"]), self.depth, B, 6 * D, 6 * D, st), "tables")
        self._final_modulation(st)
        # ---- token embedder
        concat = self.stage2 and not self.use_pe
        _lib.check(L.ga_embed_fc1(_p(s["x_in"]), self.Cin, _p(s["xyz_in"]) if concat else None, 3 if concat else 0,
                                  _p(w["fc1_w"]), _p(w["fc1_b"]), _p(s["e1"]), R, D, st), "embed_fc1")
        gemm(s["e1"], w["fc2_w"], R, D, D, epilogue(EPI_F32, bias=w["fc2_b"], out=s["xres"], ld_out=D), st)
        if self.use_pe:
            _lib.check(L.ga_xyz_posenc(_p(s["xyz_in"]), _p(s["pe"]), R, st), "xyz_pe")
            gemm(s["pe"], w["xyz_w"], R, D, 64,
                 epilogue(EPI_RESID_GATE_F32, bias=w["xyz_b"], out=s["xres"], ld_out=D, rows_per_batch=N), st)
        # ---- blocks
        for l, wb in enumerate(self.wb):
            ch = s["mod"][l].chunk(6, 1)
            for sublayer in self.block_order:
                getattr(self, sublayer)(st, l, wb, ch)
            if self.tap_blocks:
                s["taps"][l].copy_(s["xres"])
        # ---- final layer (+ CFG combine)
        _lib.check(L.ga_final_layer(_p(s["xres"]), _p(s["modf"]), _p(w["fin_w"]), _p(w["fin_b"]), _p(s["y"]), R, D,
                                    self.Cout, N, 1e-6, st), "final layer")
        if cfg_scale is not None:
            _lib.check(L.ga_cfg_combine(_p(s["y"]), _p(s["y_cfg"]), (B // 2) * N * self.Cout, cfg_scale, st), "cfg")

    @staticmethod
    def _version(t):
        try:
            return t._version
        except RuntimeError:               # inference tensors (torch.inference_mode) do not track versions
            return None

    def invalidate_context(self):
        """Forget the cached cross-attention K/V (needed only after an in-place change of a context tensor that was
        created under torch.inference_mode, where no version counter exists)."""
        self._ctx_ref = None

    def _context_is_cached(self, ctx_tok):
        # The cache holds a STRONG reference to the tensor it was computed from: while it is alive its address
        # cannot be handed to another tensor, so object identity (+ the in-place version counter) is a sound key.
        # Round 1 keyed on data_ptr(): a freed context's block is routinely recycled for the next sample's context.
        return (self._ctx_ref is not None and ctx_tok is self._ctx_ref
                and self._version(ctx_tok) == self._ctx_ver)

    def halves_identical(self, x, t, context):
        """cond | uncond halves bit-identical?  Context tensors: decided once per context object; x, t: per call."""
        key = tuple((k, id(v), self._version(v)) for k, v in sorted(context.items()) if isinstance(v, torch.Tensor))
        if self._half_ctx is None or self._half_ctx[0] != key:
            same = True
            for v in context.values():
                if isinstance(v, torch.Tensor):
                    h = v.shape[0] // 2
                    same = same and v.shape[0] % 2 == 0 and bool(torch.equal(v[:h], v[h:]))
            half = {k: (v[:v.shape[0] // 2].contiguous() if isinstance(v, torch.Tensor) else v)
                    for k, v in context.items()} if same else None
            self._half_ctx = (key, same, half, list(context.values()))      # the list pins the ids
        if not self._half_ctx[1]:
            return False
        h = x.shape[0] // 2
        if t.numel() > 1 and not bool(torch.equal(t.reshape(-1)[:h], t.reshape(-1)[h:])):
            return False
        return bool(torch.equal(x[:h], x[h:]))

    def half_context(self, context):
        return self._half_ctx[2]

    def run(self, x, t, context, cfg_scale):
        with torch.cuda.device(self.device):
            return self._run(x, t, context, cfg_scale)

    def _run(self, x, t, context, cfg_scale):
        ctx_tok, vec = context[self.ctx_key], context[self.vec_key]
        B, N, _ = x.shape
        M = ctx_tok.shape[1]
        if cfg_scale is not None and B % 2:
            raise ValueError("forward_with_cfg needs an even batch (cond | uncond)")
        if self._shape != (B, N, M):
            with torch.inference_mode(False):          # workspaces outlive this call: never inference tensors
                self._alloc(B, N, M)
        s = self.s
        if self.tap_blocks and "taps" not in s:
            with torch.inference_mode(False):
                s["taps"] = torch.zeros(self.depth, B * N, self.D, device=self.device)
        st = _launch.stream(self.device)
        s["x_in"].copy_(x.reshape(B, N, self.Cin).to(torch.float32))
        s["t_in"].copy_(t.reshape(-1).to(torch.float32).expand(B) if t.numel() == 1 else t.reshape(B).to(torch.float32))
        s["vec_in"].copy_(vec.reshape(B, self.Dc).to(torch.float32))
        if self.stage2:
            s["xyz_in"].copy_(context["fps-xyz"].reshape(B, N, 3).to(torch.float32))
        if not self._context_is_cached(ctx_tok):
            self._context_kv(st, ctx_tok.reshape(B * M, self.Dc).to(torch.float32).contiguous())
            self._ctx_ref, self._ctx_ver = ctx_tok, self._version(ctx_tok)
        gkey = (cfg_scale, self.tap_blocks)
        if self.use_graph:
            if self._graph is None or self._graph[0] != gkey:
                g, _ = _launch.capture(lambda: self._forward_launches(_launch.stream(self.device), cfg_scale), self.device)
                self._graph = (gkey, g)
            self._graph[1].replay()
        else:
            self._forward_launches(st, cfg_scale)
        out = s["y_cfg"] if cfg_scale is not None else s["y"]
        return out.clone()

    @property
    def launches_per_forward(self):
        per_block = 11
        return 8 + 2 + (2 if self.use_pe else 0) + per_block * self.depth + 1


# --------------------------------------------------------------------------
# registry (names of /root/reference/dit/dit_i23d.py:1665-1697 that map to this block type)
# --------------------------------------------------------------------------
def DiT_L_Pixelart_clay_pcd(**kw):
    return DiT_I23D_PCD_PixelArt_noclip(depth=24, use_clay_ca=True, hidden_size=1024, patch_size=1, num_heads=16,
                                        enable_rope=False, **kw)


def DiT_B_Pixelart_clay_pcd(**kw):
    return DiT_I23D_PCD_PixelArt_noclip(depth=12, use_clay_ca=True, hidden_size=768, patch_size=1, num_heads=12, **kw)


def DiT_L_Pixelart_clay_pcd_stage2(**kw):
    return DiT_I23D_PCD_PixelArt_noclip_clay_stage2(depth=24, use_clay_ca=True, hidden_size=1024, patch_size=1,
                                                    num_heads=16, use_pe_cond=True, **kw)


def DiT_B_Pixelart_clay_pcd_stage2(**kw):
    # As in the reference (dit_i23d.py:1554-1559) this entry leaves num_heads at its default of 16, i.e.
    # head_dim 48, and conditions by concatenation (use_pe_cond=False).  head_dim 48 is not supported by the
    # attention kernel, so constructing it raises ValueError; the deployed stage-2 model is the -L entry.
    return DiT_I23D_PCD_PixelArt_noclip_clay_stage2(depth=12, use_clay_ca=True, hidden_size=768, **kw)


DiT_models = {
    'DiT-PixArt-PCD-CLAY-L': DiT_L_Pixelart_clay_pcd,
    'DiT-PixArt-PCD-CLAY-B': DiT_B_Pixelart_clay_pcd,
    'DiT-PixArt-PCD-CLAY-stage2-L': DiT_L_Pixelart_clay_pcd_stage2,
    'DiT-PixArt-PCD-CLAY-stage2-B': DiT_B_Pixelart_clay_pcd_stage2,
}
