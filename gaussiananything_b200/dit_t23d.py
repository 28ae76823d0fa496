"""Mirror of the text-to-3D DiT denoisers of the reference:

  dit.dit_trilatent.DiT_PCD_PixelArt          (/root/reference/dit/dit_trilatent.py:262-332)   stage 1, xyz
  dit.dit_trilatent.DiT_PCD_PixelArt_tofeat   (/root/reference/dit/dit_trilatent.py:335-419)   stage 2, features
  block PixelArtTextCondDiTBlock              (/root/reference/dit/dit_models_xformers.py:329-376)
  FinalLayer                                  (/root/reference/dit/dit_models_xformers.py:993-1016)
  registry DiT_models                         (/root/reference/dit/dit_trilatent.py:523-536)

Same constructor arguments, attribute names and state_dict key layout (a reference checkpoint loads with
strict=True), same `forward(x, timesteps, context)` / `forward_with_cfg(x, t, context, cfg_scale)` contracts, with
context = {"caption_crossattn" [B,M,Dc], "caption_vector" [B,Dc]} (+ "fps-xyz" [B,N,3] for stage 2).  The engine is
the image DiT's (dit._DiTEngine: bf16 weight pack, workspaces, sublayer launches, CUDA graph, cached cross-attention
K/V) in the text block's order and with its modules:

  t = t_embedder(t) + cap_embedder(caption_vector);  t0 = adaLN_modulation(t);  mod = scale_shift_table + t0
  x += gate_msa * SA(RMSNorm(x) * (1 + scale_msa) + shift_msa)
  x += CA(RMSNorm(x; prenorm_ca_text), RMSNorm(context; attention_y_norm))          (no gate)
  x += gate_mlp * FFN(RMSNorm(x) * (1 + scale_mlp) + shift_mlp)
  y = Linear(LayerNorm(x) * (1 + scale) + shift),  shift, scale = Linear(SiLU(t)).chunk(2)     (FinalLayer)

Precision as in dit.py: bf16 tensor-core operands, fp32 accumulation, residual stream, norms and output.
"""
import torch
import torch.nn as nn

from . import _lib, dit
from ._launch import epilogue, gemm, ptr as _p
from ._lib import EPI_HEADS
from .dit import _CrossAttn, _FusedMLP, _Mlp, _SelfAttn, _TimestepEmbedder, _Weight, _XYZPosEmbed


class PixelArtTextCondDiTBlock(nn.Module):
    """Parameter layout of /root/reference/dit/dit_models_xformers.py:329-355 (gated SA -> CA -> gated FFN)."""

    def __init__(self, hidden_size, num_heads, mlp_ratio=4, context_dim=None, **kw):
        super().__init__()
        self.norm1 = _Weight(hidden_size)
        self.norm2 = _Weight(hidden_size)
        self.attn = _SelfAttn(hidden_size, num_heads)
        self.mlp = _FusedMLP(hidden_size, int(mlp_ratio))
        self.adaLN_modulation = None
        self.cross_attn = _CrossAttn(hidden_size, context_dim, num_heads)
        self.scale_shift_table = nn.Parameter(torch.randn(6, hidden_size) / hidden_size ** 0.5)
        self.attention_y_norm = _Weight(context_dim)
        self.prenorm_ca_text = _Weight(hidden_size)


class FinalLayer(nn.Module):
    """/root/reference/dit/dit_models_xformers.py:993-1016: LayerNorm (no affine, eps 1e-6), modulate, Linear."""

    def __init__(self, hidden_size, patch_size, out_channels):
        super().__init__()
        self.linear = nn.Linear(hidden_size, patch_size * patch_size * out_channels)
        self.adaLN_modulation = nn.Sequential(nn.SiLU(), nn.Linear(hidden_size, 2 * hidden_size))


class DiT_PCD_PixelArt(dit.DiT_I23D_PCD_PixelArt_noclip):
    def __init__(self, input_size=32, patch_size=2, in_channels=4, hidden_size=1152, depth=28, num_heads=16,
                 mlp_ratio=4, class_dropout_prob=0.1, num_classes=1000, learn_sigma=True, mixing_logit_init=-3,
                 mixed_prediction=True, context_dim=False, roll_out=False, vit_blk=None, final_layer_blk=None, **kw):
        nn.Module.__init__(self)
        if num_classes > 0:
            raise NotImplementedError("class-label conditioning is not on the text-to-3D path (the deployed models "
                                      "are built with num_classes=0)")
        if patch_size != 1:
            raise NotImplementedError("only patch_size=1 (the point-cloud registry entries) is built")
        if hidden_size % num_heads or hidden_size // num_heads != 64:
            raise ValueError("the attention kernel is specialised for head_dim 64 (got %d / %d heads)"
                             % (hidden_size, num_heads))
        if not context_dim:
            raise ValueError("the text-to-3D DiT needs context_dim (768 for the CLIP text conditioner)")
        assert roll_out
        self.depth, self.mlp_ratio, self.learn_sigma = depth, mlp_ratio, learn_sigma
        self.in_channels = in_channels
        self.out_channels = in_channels * 2 if learn_sigma else in_channels
        self.patch_size, self.num_heads, self.embed_dim = patch_size, num_heads, hidden_size
        self.roll_out, self.plane_n, self.context_dim = roll_out, 3, context_dim
        self.x_embed_in = in_channels
        self.x_embedder = _Mlp(in_channels, hidden_size, hidden_size)
        self.t_embedder = _TimestepEmbedder(hidden_size)
        self.y_embedder = None
        self.blocks = nn.ModuleList([PixelArtTextCondDiTBlock(hidden_size, num_heads, mlp_ratio, context_dim)
                                     for _ in range(depth)])
        self.final_layer = FinalLayer(hidden_size, patch_size, self.out_channels)
        self.adaLN_modulation = nn.Sequential(nn.SiLU(), nn.Linear(hidden_size, 6 * hidden_size))
        self.cap_embedder = nn.Sequential(nn.LayerNorm(context_dim), nn.Linear(context_dim, hidden_size))
        self.initialize_weights()
        self._engine = None
        self.cfg_dedup = False

    def _zero_init_linears(self):
        return (self.final_layer.linear, self.final_layer.adaLN_modulation[1], self.cap_embedder[1])

    def initialize_weights(self):
        """The reference's init (dit_models_xformers.py:1117-1159, dit_trilatent.py:171-179)."""
        for m in self.modules():
            if isinstance(m, nn.Linear):
                nn.init.xavier_uniform_(m.weight)
                if m.bias is not None:
                    nn.init.constant_(m.bias, 0)
        nn.init.normal_(self.t_embedder.mlp[0].weight, std=0.02)
        nn.init.normal_(self.t_embedder.mlp[2].weight, std=0.02)
        for lin in self._zero_init_linears():
            nn.init.constant_(lin.weight, 0)
            nn.init.constant_(lin.bias, 0)

    def randomize_zero_init_(self, std=0.02, seed=0):
        """The zero-initialised tensors would make the output identically 0 (random-weight tests and benchmarks)."""
        g = torch.Generator().manual_seed(seed)
        for lin in self._zero_init_linears() + (self.adaLN_modulation[1],):
            lin.weight.data.copy_(torch.randn(lin.weight.shape, generator=g) * std)
            lin.bias.data.copy_(torch.randn(lin.bias.shape, generator=g) * std)
        self.invalidate()
        return self

    def _new_engine(self, device):
        return _T23DEngine(self, device)


class DiT_PCD_PixelArt_tofeat(DiT_PCD_PixelArt):
    xyz_cond = True

    def __init__(self, *a, use_pe_cond=True, **kw):
        super().__init__(*a, **kw)
        self.use_pe_cond = use_pe_cond
        if use_pe_cond:
            self.xyz_pos_embed = _XYZPosEmbed(self.embed_dim)
            lin = self.xyz_pos_embed.xyz_projection
        else:
            self.x_embed_in = self.in_channels + 3
            self.x_embedder = _Mlp(self.in_channels + 3, self.embed_dim, self.embed_dim)
            lin = self.x_embedder.fc1
        nn.init.xavier_uniform_(lin.weight)
        nn.init.constant_(lin.bias, 0)


class _T23DEngine(dit._DiTEngine):
    """dit._DiTEngine with the text block: SA -> CA -> FFN, a per-block context RMSNorm before the cached K/V, and
    FinalLayer's modulation."""
    ctx_key, vec_key = "caption_crossattn", "caption_vector"
    block_order = ("self_attn", "cross_attn", "ffn")
    vec_embedder = "cap_embedder"
    ca_modules = ("cross_attn", "prenorm_ca_text")

    def _pack_block(self, b):
        return dict(super()._pack_block(b), y_w=self._f32(b.attention_y_norm.weight))

    def _pack_final_modulation(self):
        lin = self.m.final_layer.adaLN_modulation[1]
        return {"fin_ada_w": self._f32(lin.weight), "fin_ada_b": self._f32(lin.bias)}

    def _final_modulation(self, st):
        """modf [B, 2D] = final_layer.adaLN_modulation(temb) = Linear(SiLU(temb)) (FinalLayer)."""
        B, D, s, w = self._shape[0], self.D, self.s, self.w
        _lib.check(self.L.ga_linear_small(_p(s["temb"]), _p(w["fin_ada_w"]), _p(w["fin_ada_b"]), _p(s["modf"]), B, 2 * D, D,
                                          1, 0, 0, st), "final modulation")

    def _context_kv(self, st, c32):
        """Per block: RMSNorm(context; attention_y_norm) -> bf16 -> the K/V GEMM, once per context tensor."""
        B, N, M = self._shape
        s, D, H = self.s, self.D, self.H
        for l, wb in enumerate(self.wb):
            _lib.check(self.L.ga_rmsnorm_modulate(_p(c32), _p(wb["y_w"]), None, None, 0, M, _p(s["ctx"]), B * M, self.Dc,
                                                  1e-5, st), "attention_y_norm")
            e = epilogue(EPI_HEADS, k=s["kc"][l], vt=s["vtc"][l], kn_w=wb["cak_n"], heads=H, first_part=1,
                         tok_pitch=self.Mp, rows_per_batch=M)
            gemm(s["ctx"], wb["cakv_w"], B * M, 2 * D, self.Dc, e, st)


# --------------------------------------------------------------------------
# registry (/root/reference/dit/dit_trilatent.py:479-536, the point-cloud entries)
# --------------------------------------------------------------------------
def DiT_PCD_B(**kw):
    return DiT_PCD_PixelArt(depth=12, hidden_size=768, patch_size=1, num_heads=12, **kw)


def DiT_PCD_L(**kw):
    return DiT_PCD_PixelArt(depth=24, hidden_size=1024, patch_size=1, num_heads=16, **kw)


def DiT_PCD_B_tofeat(**kw):
    return DiT_PCD_PixelArt_tofeat(depth=12, hidden_size=768, patch_size=1, num_heads=12, **kw)


def DiT_PCD_L_tofeat(**kw):
    return DiT_PCD_PixelArt_tofeat(depth=24, hidden_size=1024, patch_size=1, num_heads=16, **kw)


def DiT_PCD_XL_tofeat(**kw):
    # D 1152 with 16 heads is head_dim 72, which the attention kernel does not support: constructing it raises
    # ValueError.  The deployed stage-2 text model is the -L entry.
    return DiT_PCD_PixelArt_tofeat(depth=28, hidden_size=1152, patch_size=1, num_heads=16, **kw)


DiT_models = {
    'DiT-PCD-B': DiT_PCD_B,
    'DiT-PCD-L': DiT_PCD_L,
    'DiT-PCD-B-stage2-xyz2feat': DiT_PCD_B_tofeat,
    'DiT-PCD-L-stage2-xyz2feat': DiT_PCD_L_tofeat,
    'DiT-PCD-XL-stage2-xyz2feat': DiT_PCD_XL_tofeat,
}
