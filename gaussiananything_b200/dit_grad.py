"""Training forward and backward of the image-to-3D DiT block on the library's kernels (include/ga_b200.h Part 14).

ImageCondDiTBlockPixelArtRMSNormClayLRM.forward (the reference's dit/dit_models_xformers.py:765-787), the unit that
repeats 24 times in DiT-L:

    shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp = scale_shift_table + t     (mod [B, 6, D])
    x1 = x  + cross_attn_dino(prenorm_ca_dino(x), context)                     (q/k RMSNorm per head)
    x2 = x1 + gate_msa * attn(norm1(x1) * (1 + scale_msa) + shift_msa)         (q/k RMSNorm per head)
    y  = x2 + gate_mlp * mlp(norm2(x2) * (1 + scale_mlp) + shift_mlp)          (FusedMLP, exact GELU)

    from gaussiananything_b200 import dit_grad
    y = dit_grad.block_forward(block, x, t, context)      # x [B, N, D], t [B, 6 D], context [B, M, Dc]
    y.sum().backward()                                    # x.grad, t.grad, context.grad and every parameter's grad

The forward keeps what the backward reads: the fp32 residual stream x, x1, x2, the fp32 outputs a2 = proj(...) and
a3 = fc2(...) the gates multiply, every bf16 GEMM and attention operand, the attentions' log-sum-exp and fc1's
pre-activation.  The backward runs the chain in reverse on the Part 12 attention backward, the Part 13 dgrad, wgrad
and bias-gradient GEMMs and the Part 14 row kernels, forming each gradient only when something needs it.  Under
no_grad, or when nothing requires grad, nothing is saved.

GEMM and attention operands are bf16, norms, residuals and gates fp32 (the reference trains under bf16 autocast).
Gradients come back in their tensor's dtype.  There is no CPU fallback, no RoPE and no head_dim other than 64.
"""
import ctypes as C
import math

import torch

from . import _lib
from ._launch import epilogue, gemm, ptr, stream
from ._lib import EPI_RESID_GATE_F32
from .attention import _backward as _attention_bwd, _forward as _attention
from .mlp import _bgrad, _dgrad, _fc1, _forward_linear, _pack, _wgrad

__all__ = ["block_forward", "model_forward"]

_BF16, _F32 = torch.bfloat16, torch.float32
_EPS = 1e-5
_SCALE = 1.0 / math.sqrt(64.0)
_NPARAM = 21


def block_parameters(block):
    """The 21 parameters of the block in the order the autograd function takes them."""
    ca, sa, mlp = block.cross_attn_dino, block.attn, block.mlp.mlp
    return (block.scale_shift_table, block.prenorm_ca_dino.weight, block.norm1.weight, block.norm2.weight,
            ca.to_q.weight, ca.to_k.weight, ca.to_v.weight, ca.q_norm.weight, ca.k_norm.weight,
            ca.to_out[0].weight, ca.to_out[0].bias,
            sa.qkv.weight, sa.qkv.bias, sa.q_norm.weight, sa.k_norm.weight, sa.proj.weight, sa.proj.bias,
            mlp[0].weight, mlp[1].bias, mlp[2].weight, mlp[3].bias)


def _f32(t):
    return t.detach().to(_F32).contiguous()


def _at(t, elems):
    """The address `elems` elements into t (a modulation chunk of mod [B, 6 D])."""
    return C.c_void_p(t.data_ptr() + elems * t.element_size())


def _heads(m, B, N, parts, j):
    """Part j of a "(K H D)" bf16 matrix m [B N, parts H 64] as the [B, N, H, 64] view the attention reads."""
    return m.view(B, N, parts, -1, 64)[:, :, j]


def _qk_norm(src, ld_in, w0, w1, rows, heads, parts):
    out = torch.empty((rows, 64 * heads * parts), dtype=_BF16, device=src.device)
    _lib.check(_lib.lib().ga_dit_qk_norm_fwd_bf16(ptr(src), ld_in, ptr(out), out.shape[1], ptr(w0), ptr(w1), rows,
                                                  heads, parts, _EPS, stream(src.device)), "ga_dit_qk_norm_fwd_bf16")
    return out


def _qk_norm_bwd(src, ld_in, d, ld_d, w0, w1, rows, heads, parts):
    """Overwrites the attention's dq/dk in d with the pre-norm gradient; returns the weight-gradient partials."""
    L = _lib.lib()
    part = torch.empty((parts, L.ga_dit_grad_partials(rows, rows), 64), dtype=_F32, device=src.device)
    _lib.check(L.ga_dit_qk_norm_bwd_bf16(ptr(src), ld_in, ptr(d), ld_d, ptr(d), ld_d, ptr(w0), ptr(w1), ptr(part),
                                         rows, heads, parts, _EPS, stream(src.device)), "ga_dit_qk_norm_bwd_bf16")
    return part


def _reduce(part, groups, cols):
    """[groups, cols] = the partials part [groups, P, cols] added in order."""
    out = torch.empty((groups, cols), dtype=_F32, device=part.device)
    _lib.check(_lib.lib().ga_dit_grad_reduce(ptr(part), ptr(out), groups, part.numel() // (groups * cols), cols,
                                             stream(part.device)), "ga_dit_grad_reduce")
    return out


def _gate_residual(x, a, gate, x_out, w=None, shift=None, scale=None, h=None, N=1, D=1):
    R = x.shape[0]
    _lib.check(_lib.lib().ga_dit_gate_residual(ptr(x), ptr(a), gate, 6 * D, ptr(x_out), ptr(w), shift, scale, 6 * D,
                                               ptr(h), N, R, D, _EPS, stream(x.device)), "ga_dit_gate_residual")


def _forward(x, t, ctx, params, keep):
    """The block on prepared operands; returns (y fp32 [B N, D], the saved state or None)."""
    (sst, pre_w, n1_w, n2_w, q_w, k_w, v_w, caqn, cakn, o_w, o_b, qkv_w, qkv_b, qn, kn, p_w, p_b,
     w1, b1, w2, b2) = params
    B, N, D = x.shape
    M, Dc = ctx.shape[1], ctx.shape[2]
    H, R, RM = D // 64, B * N, B * M
    dev = x.device
    L, st = _lib.lib(), stream(dev)
    xf = x.detach().to(_F32).contiguous().view(R, D)
    tf = t.detach().to(_F32).contiguous().view(B, 6 * D)
    ctxb = ctx.detach().to(_BF16).contiguous().view(RM, Dc)
    wq, wkv, wo, wqkv, wp, w1b, w2b = (_pack(q_w), _pack(torch.cat([k_w.detach(), v_w.detach()])), _pack(o_w),
                                       _pack(qkv_w), _pack(p_w), _pack(w1), _pack(w2))
    f = [_f32(p) for p in (sst, pre_w, n1_w, n2_w, caqn, cakn, o_b, qkv_b, qn, kn, p_b, b1, b2)]
    sstf, pre_f, n1_f, n2_f, caqn_f, cakn_f, o_bf, qkv_bf, qn_f, kn_f, p_bf, b1f, b2f = f
    mod = torch.empty((B, 6 * D), dtype=_F32, device=dev)
    _lib.check(L.ga_add_tables(ptr(sstf), ptr(tf), ptr(mod), 1, B, 6 * D, 6 * D, st), "ga_add_tables")
    ch = lambda j: _at(mod, j * D)
    # cross-attention on the context (pre-norm, residual)
    h0 = torch.empty((R, D), dtype=_BF16, device=dev)
    _lib.check(L.ga_rmsnorm_modulate(ptr(xf), ptr(pre_f), None, None, 0, N, ptr(h0), R, D, _EPS, st),
               "ga_rmsnorm_modulate")
    qc = _forward_linear(h0, wq, None, _BF16)
    kv = _forward_linear(ctxb, wkv, None, _BF16)                       # [B M, 2 D]: k | v
    qcn = _qk_norm(qc, D, caqn_f, None, R, H, 1)
    kcn = _qk_norm(kv, 2 * D, cakn_f, None, RM, H, 1)
    o_ca, lse_ca = _attention(qcn.view(B, N, H, 64), kcn.view(B, M, H, 64), _heads(kv, B, M, 2, 1), _SCALE)
    a1 = _forward_linear(o_ca.view(R, D), wo, o_bf, _F32)
    x1, h1 = torch.empty_like(xf), torch.empty_like(h0)
    _gate_residual(xf, a1, None, x1, n1_f, ch(0), ch(1), h1, N, D)
    # gated self-attention
    qkv = _forward_linear(h1, wqkv, qkv_bf, _BF16)                      # [B N, 3 D]: q | k | v
    qkn = _qk_norm(qkv, 3 * D, qn_f, kn_f, R, H, 2)
    o_sa, lse_sa = _attention(_heads(qkn, B, N, 2, 0), _heads(qkn, B, N, 2, 1), _heads(qkv, B, N, 3, 2), _SCALE)
    a2 = _forward_linear(o_sa.view(R, D), wp, p_bf, _F32)
    x2, h2 = torch.empty_like(xf), torch.empty_like(h0)
    _gate_residual(x1, a2, ch(2), x2, n2_f, ch(3), ch(4), h2, N, D)
    # gated FFN
    hid, z = _fc1(h2, w1b, b1f, keep_pre=keep)
    a3 = _forward_linear(hid, w2b, b2f, _F32)
    y = torch.empty_like(xf)
    _gate_residual(x2, a3, ch(5), y, N=N, D=D)
    if not keep:
        return y, None
    saved = (xf, mod, h0, ctxb, qc, kv, qcn, kcn, o_ca, lse_ca, x1, h1, qkv, qkn, o_sa, lse_sa, a2, x2, h2, z, hid,
             a3, wq, wkv, wo, wqkv, wp, w1b, w2b, pre_f, n1_f, n2_f, caqn_f, cakn_f, qn_f, kn_f)
    return y, saved


class _DiTBlock(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, t, context, *params):
        with torch.cuda.device(x.device):
            y, saved = _forward(x, t, context, params, keep=True)
        # the parameters themselves are saved too, so that changing one in place before backward raises
        ctx.save_for_backward(*saved, *params)
        ctx.meta = (x.shape, x.dtype, t.shape, t.dtype, context.shape, context.dtype)
        return y.view(x.shape).to(x.dtype)

    @staticmethod
    def backward(ctx, gy):
        if torch.is_grad_enabled():
            raise RuntimeError("dit_grad: double backward (create_graph=True) is not supported")
        with torch.cuda.device(gy.device):
            return _backward(ctx, gy)


def _backward(ctx, gy):
    saved = ctx.saved_tensors
    (xf, mod, h0, ctxb, qc, kv, qcn, kcn, o_ca, lse_ca, x1, h1, qkv, qkn, o_sa, lse_sa, a2, x2, h2, z, hid, a3,
     wq, wkv, wo, wqkv, wp, w1b, w2b, pre_f, n1_f, n2_f, caqn_f, cakn_f, qn_f, kn_f) = saved[:-_NPARAM]
    params = saved[-_NPARAM:]
    x_shape, x_dtype, t_shape, t_dtype, c_shape, c_dtype = ctx.meta
    need = ctx.needs_input_grad
    nx, nt, nc = need[:3]
    (n_sst, n_pre, n_n1, n_n2, n_q, n_k, n_v, n_cqn, n_ckn, n_ow, n_ob, n_qkvw, n_qkvb, n_qn, n_kn, n_pw, n_pb,
     n_w1, n_b1, n_w2, n_b2) = need[3:]
    B, N, D = x_shape
    M, Dc = c_shape[1], c_shape[2]
    H, R, RM = D // 64, B * N, B * M
    dev = xf.device
    L, st = _lib.lib(), stream(dev)
    n_mod = nt or n_sst
    q_side = nx or n_pre or n_q or n_cqn                 # the gradient of the cross-attention's query
    kv_side = nc or n_k or n_v or n_ckn                   # ... and of its keys and values
    need_dx1 = q_side or kv_side or n_ow or n_ob
    need_dx2 = need_dx1 or n_mod or n_n1 or n_qkvw or n_qkvb or n_qn or n_kn or n_pw or n_pb
    need_dh2 = need_dx2 or n_n2
    P = L.ga_dit_grad_partials(R, N)
    grads = [None] * (3 + _NPARAM)
    dy = gy.reshape(R, D).to(_F32).contiguous()
    pmod = torch.empty((P, 6 * D), dtype=_F32, device=dev)              # partials of dt, chunk by chunk
    pnorm = torch.empty((3, P, D), dtype=_F32, device=dev)              # prenorm, norm1, norm2 weight partials

    def gate_bwd(d, a, j):
        da = torch.empty((R, D), dtype=_BF16, device=dev)
        _lib.check(L.ga_dit_gate_bwd(ptr(d), ptr(a), _at(mod, j * D), 6 * D, ptr(da), _at(pmod, j * D), 6 * D, N, R,
                                     D, st), "ga_dit_gate_bwd")
        return da

    def norm_bwd(dh, xin, w, i, j, dx_in, want_dx):
        dx = torch.empty_like(xf) if want_dx else None
        mods = (_at(mod, (j + 1) * D), _at(pmod, j * D), _at(pmod, (j + 1) * D)) if j is not None else (None,) * 3
        _lib.check(L.ga_dit_rmsnorm_bwd(ptr(dh), ptr(xin), ptr(w), mods[0], 6 * D, ptr(dx_in if want_dx else None),
                                        ptr(dx), ptr(pnorm[i]),
                                        mods[1], mods[2], 6 * D, N, R, D, _EPS, st), "ga_dit_rmsnorm_bwd")
        return dx

    # ---- gated FFN: y = x2 + gate_mlp a3
    da3 = gate_bwd(dy, a3, 5)
    if n_b2:
        grads[23] = _bgrad(da3)
    if n_w2:
        grads[22] = _wgrad(da3, hid)
    dx2 = None
    if n_w1 or n_b1 or need_dh2:
        dz = _dgrad(da3, w2b, z=z)
        if n_b1:
            grads[21] = _bgrad(dz)
        if n_w1:
            grads[20] = _wgrad(dz, h2)
        if need_dh2:
            dx2 = norm_bwd(_dgrad(dz, w1b, f32=True), x2, n2_f, 2, 3, dy, need_dx2)
    # ---- gated self-attention: x2 = x1 + gate_msa a2
    dx1 = None
    if need_dx2:
        da2 = gate_bwd(dx2, a2, 2)
        if n_pb:
            grads[19] = _bgrad(da2)
        if n_pw:
            grads[18] = _wgrad(da2, o_sa.view(R, D))
        if need_dx1 or n_mod or n_n1 or n_qkvw or n_qkvb or n_qn or n_kn:
            do = _dgrad(da2, wp).view(B, N, H, 64)
            dqkv = torch.empty((R, 3 * D), dtype=_BF16, device=dev)
            _attention_bwd(_heads(qkn, B, N, 2, 0), _heads(qkn, B, N, 2, 1), _heads(qkv, B, N, 3, 2), o_sa, lse_sa,
                           do, _heads(dqkv, B, N, 3, 0), _heads(dqkv, B, N, 3, 1), _heads(dqkv, B, N, 3, 2), _SCALE)
            pqk = _qk_norm_bwd(qkv, 3 * D, dqkv, 3 * D, qn_f, kn_f, R, H, 2)
            if n_qn or n_kn:
                dqk = _reduce(pqk, 2, 64)
                grads[16], grads[17] = dqk[0], dqk[1]
            if n_qkvb:
                grads[15] = _bgrad(dqkv)
            if n_qkvw:
                grads[14] = _wgrad(dqkv, h1)
            if need_dx1 or n_mod or n_n1:
                dx1 = norm_bwd(_dgrad(dqkv, wqkv, f32=True), x1, n1_f, 1, 0, dx2, need_dx1)
    # ---- cross-attention: x1 = x + to_out(attention)
    dx = None
    if need_dx1:
        da1 = torch.empty((R, D), dtype=_BF16, device=dev)
        _lib.check(L.ga_f32_to_bf16(ptr(dx1), ptr(da1), R * D, st), "ga_f32_to_bf16")
        if n_ob:
            grads[13] = _bgrad(da1)
        if n_ow:
            grads[12] = _wgrad(da1, o_ca.view(R, D))
        if q_side or kv_side:
            do = _dgrad(da1, wo).view(B, N, H, 64)
            dq = torch.empty((R, D), dtype=_BF16, device=dev) if q_side else None
            dkv = torch.empty((RM, 2 * D), dtype=_BF16, device=dev) if kv_side else None
            _attention_bwd(qcn.view(B, N, H, 64), kcn.view(B, M, H, 64), _heads(kv, B, M, 2, 1), o_ca, lse_ca, do,
                           dq.view(B, N, H, 64) if q_side else None,
                           _heads(dkv, B, M, 2, 0) if kv_side else None,
                           _heads(dkv, B, M, 2, 1) if kv_side else None, _SCALE)
            if q_side:
                pq = _qk_norm_bwd(qc, D, dq, D, caqn_f, None, R, H, 1)
                if n_cqn:
                    grads[10] = _reduce(pq, 1, 64)[0]
                if n_q:
                    grads[7] = _wgrad(dq, h0)
                if nx or n_pre:
                    dx = norm_bwd(_dgrad(dq, wq, f32=True), xf, pre_f, 0, None, dx1, nx)
            if kv_side:
                pk = _qk_norm_bwd(kv, 2 * D, dkv, 2 * D, cakn_f, None, RM, H, 1)
                if n_ckn:
                    grads[11] = _reduce(pk, 1, 64)[0]
                if n_k or n_v:
                    dwkv = _wgrad(dkv, ctxb)
                    grads[8], grads[9] = dwkv[:D], dwkv[D:]
                if nc:
                    grads[2] = _dgrad(dkv, wkv, f32=True).view(c_shape).to(c_dtype)
    if nx:
        grads[0] = dx.view(x_shape).to(x_dtype)
    # ---- norm weights and the modulation
    for i, (slot, wanted) in enumerate(((4, n_pre), (5, n_n1), (6, n_n2))):
        if wanted:
            grads[slot] = _reduce(pnorm[i], 1, D)[0]
    if n_mod:
        dt = _reduce(pmod, B, 6 * D)                                     # [B, 6 D]
        if nt:
            grads[1] = dt.view(t_shape).to(t_dtype)
        if n_sst:
            grads[3] = _reduce(dt, 1, 6 * D).view(6, D)
    for i, p in enumerate(params):
        g = grads[3 + i]
        if g is not None:
            grads[3 + i] = g.to(p.dtype) if g.shape == p.shape else g.reshape(p.shape).to(p.dtype)
    return tuple(grads)


def _check(block, x, t, context, freqs_cis):
    if freqs_cis is not None:
        raise NotImplementedError("ImageCondDiTBlockPixelArtRMSNormClayLRM: RoPE (freqs_cis) is not supported")
    for name, v in (("x", x), ("t", t), ("dino_spatial_token", context)):
        if not isinstance(v, torch.Tensor):
            raise TypeError("ImageCondDiTBlockPixelArtRMSNormClayLRM: %s must be a tensor" % name)
        if v.dtype not in (torch.float32, torch.bfloat16, torch.float16):
            raise TypeError("ImageCondDiTBlockPixelArtRMSNormClayLRM: %s must be fp32, bf16 or fp16, got %s"
                            % (name, v.dtype))
    D = block.scale_shift_table.shape[1]
    heads = block.num_heads
    if D % heads or D // heads != 64:
        raise NotImplementedError("ImageCondDiTBlockPixelArtRMSNormClayLRM: head_dim %s is not supported (64 only)"
                                  % (D / heads,))
    if x.dim() != 3 or x.shape[2] != D or x.shape[0] < 1 or x.shape[1] < 1:
        raise ValueError("ImageCondDiTBlockPixelArtRMSNormClayLRM: x must be [B, N, %d], got %s" % (D, tuple(x.shape)))
    B = x.shape[0]
    if t.numel() != B * 6 * D:
        raise ValueError("ImageCondDiTBlockPixelArtRMSNormClayLRM: t must hold [B, 6 D] = %d values, got %s"
                         % (B * 6 * D, tuple(t.shape)))
    Dc = block.cross_attn_dino.to_k.weight.shape[1]
    if context.dim() != 3 or context.shape[0] != B or context.shape[2] != Dc or context.shape[1] < 1:
        raise ValueError("ImageCondDiTBlockPixelArtRMSNormClayLRM: dino_spatial_token must be [%d, M, %d], got %s"
                         % (B, Dc, tuple(context.shape)))
    if D > 1024 or Dc % 8:
        raise NotImplementedError("ImageCondDiTBlockPixelArtRMSNormClayLRM: hidden size %d > 1024 or context width "
                                  "%d not a multiple of 8" % (D, Dc))
    params = block_parameters(block)
    if not (x.is_cuda and t.is_cuda and context.is_cuda and all(p.is_cuda for p in params)):
        raise RuntimeError("ImageCondDiTBlockPixelArtRMSNormClayLRM needs CUDA tensors (there is no CPU fallback)")
    if any(v.device != x.device for v in (t, context) + params):
        raise ValueError("ImageCondDiTBlockPixelArtRMSNormClayLRM: inputs and parameters are on different devices")
    return params


def block_forward(block, x, t, context, freqs_cis=None):
    """The block's forward with a backward: x [B, N, D] (the residual stream), t [B, 6 D] (the shared adaLN output),
    context [B, M, Dc] (the DINOv2 tokens).  Returns y [B, N, D] in x's dtype."""
    params = _check(block, x, t, context, freqs_cis)
    if torch.is_grad_enabled() and any(v.requires_grad for v in (x, t, context) + params):
        return _DiTBlock.apply(x, t, context, *params)
    with torch.cuda.device(x.device):
        y, _ = _forward(x, t, context, params, keep=False)
    return y.view(x.shape).to(x.dtype)


# ---- the whole model: stem -> blocks -> head (include/ga_b200.h Part 15) ---------------------------------------------
#
# model_forward(model, x, timesteps, context) is DiT_I23D_PCD_PixelArt_noclip.forward (the reference's
# dit/dit_i23d.py:511-567, stage 2 :707-750) with a backward, in three autograd pieces:
#   stem   (x, img_vector, the stem parameters) -> (xres [B, N, D] the residual stream, t0 [B, 6 D], temb [B, D])
#   blocks _DiTBlock per block, each fed the same t0, so autograd adds their dt
#   head   (xres, temb, the final layer's parameters) -> y [B, N, out_channels]
# The stem's backward gets dt0 from the blocks and dtemb from the head.  timesteps and context["fps-xyz"] are
# constants.  The forward runs the launches of the inference engine (dit._DiTEngine._forward_launches) with the same
# precision: the B-row stem in fp32, the token embedder's GEMMs on bf16 operands.

_SMALL_ROWS = 16                                            # ga_linear_small's row limit


def _linear_small(x, W, b, y, act_in=0, accumulate=0):
    """y [B, N] (+)= act(x) W^T + b over 16-row chunks, any B (fp32 ga_linear_small)."""
    B, K = x.shape
    N = W.shape[0]
    for r0 in range(0, B, _SMALL_ROWS):
        n = min(_SMALL_ROWS, B - r0)
        _lib.check(_lib.lib().ga_linear_small(_at(x, r0 * K), ptr(W), ptr(b), _at(y, r0 * N), n, N, K, act_in, 0,
                                              accumulate, stream(x.device)), "ga_linear_small")


def _linear_small_bwd(x, act_in, W, dy, want_w, want_b, want_x, dx_in=None):
    """(dW, db, dx) of y = act(x) W^T + b for dy [B, N]; dx = dx_in + act'(x) (dy W).  None where not wanted."""
    B, K = x.shape
    N = W.shape[0]
    L, dev = _lib.lib(), x.device
    dW = torch.empty((N, K), dtype=_F32, device=dev) if want_w else None
    db = torch.empty(N, dtype=_F32, device=dev) if want_b else None
    dx = part = None
    if want_x:
        dx = torch.empty((B, K), dtype=_F32, device=dev)
        part = torch.empty((L.ga_dit_grad_partials(N, N), B, K), dtype=_F32, device=dev)
    if want_w or want_b or want_x:
        _lib.check(L.ga_dit_linear_small_bwd(ptr(x), act_in, ptr(W), ptr(dy), ptr(dW), ptr(db), ptr(part),
                                             ptr(dx_in if want_x else None), ptr(dx), B, N, K, stream(dev)),
                   "ga_dit_linear_small_bwd")
    return dW, db, dx


def stem_parameters(model):
    """The stem's parameters in the order the autograd function takes them."""
    t, v, a, e = model.t_embedder.mlp, model.pooled_vec_embedder, model.adaLN_modulation[1], model.x_embedder
    p = (t[0].weight, t[0].bias, t[2].weight, t[2].bias, v[0].weight, v[0].bias, v[1].weight, v[1].bias,
         a.weight, a.bias, e.fc1.weight, e.fc1.bias, e.fc2.weight, e.fc2.bias)
    if _uses_pe(model):
        p += (model.xyz_pos_embed.xyz_projection.weight, model.xyz_pos_embed.xyz_projection.bias)
    return p


def head_parameters(model):
    f = model.final_layer
    return (f.scale_shift_table, f.linear.weight, f.linear.bias)


def _uses_pe(model):
    return bool(model.xyz_cond and model.use_pe_cond)


def _stem_forward(x, vec, t, xyz, params, keep):
    """(xres fp32 [B N, D], t0 [B, 6 D], temb [B, D], the saved state or None)."""
    (t0_w, t0_b, t2_w, t2_b, ln_w, ln_b, v_w, v_b, a_w, a_b, f1_w, f1_b, f2_w, f2_b) = params[:14]
    use_pe = len(params) == 16
    B, N, Cin = x.shape
    D, Dc, R = t2_w.shape[0], vec.shape[-1], B * N
    dev = x.device
    L, st = _lib.lib(), stream(dev)
    f = [_f32(p) for p in (t0_w, t0_b, t2_w, t2_b, ln_w, ln_b, v_w, v_b, a_w, a_b, f1_w, f1_b, f2_b)]
    t0_wf, t0_bf, t2_wf, t2_bf, ln_wf, ln_bf, v_wf, v_bf, a_wf, a_bf, f1_wf, f1_bf, f2_bf = f
    f2_wb = _pack(f2_w)
    tf = t.detach().to(_F32).reshape(-1).expand(B).contiguous() if t.numel() == 1 else _f32(t).view(B)
    sinus = torch.empty((B, 256), dtype=_F32, device=dev)
    _lib.check(L.ga_timestep_sinusoid(ptr(tf), ptr(sinus), B, 256, st), "ga_timestep_sinusoid")
    a1 = torch.empty((B, D), dtype=_F32, device=dev)                   # t_embedder's pre-SiLU activation
    _linear_small(sinus, t0_wf, t0_bf, a1)
    temb = torch.empty((B, D), dtype=_F32, device=dev)
    _linear_small(a1, t2_wf, t2_bf, temb, act_in=1)
    vf = _f32(vec).view(B, Dc)
    vln = torch.empty((B, Dc), dtype=_F32, device=dev)
    _lib.check(L.ga_layernorm_rows(ptr(vf), ptr(ln_wf), ptr(ln_bf), ptr(vln), B, Dc, 1e-5, st), "ga_layernorm_rows")
    _linear_small(vln, v_wf, v_bf, temb, accumulate=1)
    t0 = torch.empty((B, 6 * D), dtype=_F32, device=dev)
    _linear_small(temb, a_wf, a_bf, t0, act_in=1)
    # token embedder (+ the xyz conditioning of stage 2)
    xf = _f32(x).view(R, Cin)
    xyzf = _f32(xyz).view(R, 3) if xyz is not None else None
    concat = xyz is not None and not use_pe
    e1 = torch.empty((R, D), dtype=_BF16, device=dev)
    _lib.check(L.ga_embed_fc1(ptr(xf), Cin, ptr(xyzf) if concat else None, 3 if concat else 0, ptr(f1_wf), ptr(f1_bf),
                              ptr(e1), R, D, st), "ga_embed_fc1")
    xres = _forward_linear(e1, f2_wb, f2_bf, _F32)
    pe = xyz_wb = None
    if use_pe:
        pe = torch.empty((R, 64), dtype=_BF16, device=dev)
        _lib.check(L.ga_xyz_posenc(ptr(xyzf), ptr(pe), R, st), "ga_xyz_posenc")
        xyz_wb = torch.zeros((D, 64), dtype=_BF16, device=dev)           # K padded 63 -> 64, the padded column 0
        xyz_wb[:, :63] = params[14].detach()
        gemm(pe, xyz_wb, R, D, 64, epilogue(EPI_RESID_GATE_F32, bias=_f32(params[15]), out=xres, ld_out=D,
                                            rows_per_batch=N), st)
    if not keep:
        return xres, t0, temb, None
    saved = (sinus, a1, vf, vln, temb, xf, e1, f2_wb, t0_wf, t2_wf, ln_wf, v_wf, a_wf, f1_wf, f1_bf)
    saved += ((xyzf,) if xyz is not None else ()) + ((pe,) if use_pe else ())
    return xres, t0, temb, saved


class _DiTStem(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, vec, t, xyz, *params):
        with torch.cuda.device(x.device):
            xres, t0, temb, saved = _stem_forward(x, vec, t, xyz, params, keep=True)
        ctx.save_for_backward(*saved, *params)
        ctx.meta = (x.shape, x.dtype, vec.shape, vec.dtype, xyz is not None, len(params))
        return xres.view(x.shape[0], x.shape[1], -1), t0, temb

    @staticmethod
    def backward(ctx, dxres, dt0, dtemb):
        if torch.is_grad_enabled():
            raise RuntimeError("dit_grad: double backward (create_graph=True) is not supported")
        with torch.cuda.device(dxres.device):
            return _stem_backward(ctx, dxres, dt0, dtemb)


def _stem_backward(ctx, dxres, dt0, dtemb):
    x_shape, x_dtype, v_shape, v_dtype, stage2, nparam = ctx.meta
    use_pe = nparam == 16
    saved = ctx.saved_tensors
    params = saved[-nparam:]
    sinus, a1, vf, vln, temb, xf, e1, f2_wb, t0_wf, t2_wf, ln_wf, v_wf, a_wf, f1_wf, f1_bf = saved[:15]
    xyzf = saved[15] if stage2 else None
    pe = saved[16] if use_pe else None
    need = ctx.needs_input_grad
    nx, nvec = need[0], need[1]
    n = need[4:] + (False, False)
    (n_t0w, n_t0b, n_t2w, n_t2b, n_lnw, n_lnb, n_vw, n_vb, n_aw, n_ab, n_f1w, n_f1b, n_f2w, n_f2b, n_xw, n_xb) = n[:16]
    B, N, Cin = x_shape
    D, R = temb.shape[1], B * N
    dev = temb.device
    L, st = _lib.lib(), stream(dev)
    grads = [None] * (4 + nparam)
    # ---- token embedder: xres = fc2(e1) (+ xyz projection)
    fc1_side = nx or n_f1w or n_f1b
    if fc1_side or n_f2w or n_f2b or n_xw or n_xb:
        g = torch.empty((R, D), dtype=_BF16, device=dev)
        _lib.check(L.ga_f32_to_bf16(ptr(dxres.to(_F32).contiguous()), ptr(g), R * D, st), "ga_f32_to_bf16")
        if n_xw:
            grads[4 + 14] = _wgrad(g, pe)[:, :63].contiguous()         # the padded column carries no parameter
        if n_f2w:
            grads[4 + 12] = _wgrad(g, e1)
        if n_f2b or n_xb:
            db = _bgrad(g)                               # fc2 and the xyz projection share their output's bias sum
            if n_f2b:
                grads[4 + 13] = db
            if n_xb:
                grads[4 + 15] = db.clone() if n_f2b else db              # one tensor per .grad
        if fc1_side:
            de1 = _dgrad(g, f2_wb, f32=True)
            concat = stage2 and not use_pe
            K = Cin + (3 if concat else 0)
            P = L.ga_dit_grad_partials(R, R)
            pw, pb = (torch.empty((P, D * K), dtype=_F32, device=dev), torch.empty((P, D), dtype=_F32, device=dev))
            dxin = torch.empty((R, Cin), dtype=_F32, device=dev) if nx else None
            _lib.check(L.ga_dit_embed_fc1_bwd(ptr(xf), Cin, ptr(xyzf) if concat else None, 3 if concat else 0,
                                              ptr(f1_wf), ptr(f1_bf), ptr(de1), ptr(pw), ptr(pb), ptr(dxin), R, D, st),
                       "ga_dit_embed_fc1_bwd")
            if n_f1w:
                grads[4 + 10] = _reduce(pw, 1, D * K).view(D, K)
            if n_f1b:
                grads[4 + 11] = _reduce(pb, 1, D)[0]
            if nx:
                grads[0] = dxin.view(x_shape).to(x_dtype)
    # ---- vector path: t0 = ada(silu(temb)), temb = t2(silu(a1)) + vec1(LN(vec)), a1 = t0(sinus)
    up_t = n_t0w or n_t0b or n_t2w or n_t2b
    up_v = nvec or n_lnw or n_lnb or n_vw or n_vb
    dt0 = dt0.to(_F32).contiguous()
    dtemb = dtemb.to(_F32).contiguous()
    grads[4 + 8], grads[4 + 9], dtemb = _linear_small_bwd(temb, 1, a_wf, dt0, n_aw, n_ab, up_t or up_v, dx_in=dtemb)
    if up_t:
        grads[4 + 2], grads[4 + 3], da1 = _linear_small_bwd(a1, 1, t2_wf, dtemb, n_t2w, n_t2b, n_t0w or n_t0b)
        if n_t0w or n_t0b:
            grads[4 + 0], grads[4 + 1], _ = _linear_small_bwd(sinus, 0, t0_wf, da1, n_t0w, n_t0b, False)
    if up_v:
        grads[4 + 6], grads[4 + 7], dvln = _linear_small_bwd(vln, 0, v_wf, dtemb, n_vw, n_vb, nvec or n_lnw or n_lnb)
        if nvec or n_lnw or n_lnb:
            Dc = vf.shape[1]
            dvec = torch.empty_like(vf) if nvec else None
            dw = torch.empty(Dc, dtype=_F32, device=dev) if n_lnw else None
            db = torch.empty(Dc, dtype=_F32, device=dev) if n_lnb else None
            _lib.check(L.ga_dit_layernorm_rows_bwd(ptr(vf), ptr(ln_wf), ptr(dvln), ptr(dvec), ptr(dw), ptr(db), B, Dc,
                                                   1e-5, st), "ga_dit_layernorm_rows_bwd")
            grads[4 + 4], grads[4 + 5] = dw, db
            if nvec:
                grads[1] = dvec.view(v_shape).to(v_dtype)
    for i, p in enumerate(params):
        g = grads[4 + i]
        if g is not None:
            grads[4 + i] = g.view(p.shape).to(p.dtype)
    return tuple(grads)


def _head_forward(xres, temb, params, N, keep):
    table, W, b = params
    R, D = xres.shape
    B, Cout = temb.shape[0], W.shape[0]
    dev = xres.device
    L, st = _lib.lib(), stream(dev)
    tf, Wf, bf = _f32(table), _f32(W), _f32(b)
    tembf = temb.detach().to(_F32).contiguous()
    modf = torch.empty((B, 2 * D), dtype=_F32, device=dev)
    _lib.check(L.ga_add_tables(ptr(tf), ptr(tembf), ptr(modf), 1, B, 2 * D, D, st), "ga_add_tables")
    y = torch.empty((R, Cout), dtype=_F32, device=dev)
    _lib.check(L.ga_final_layer(ptr(xres), ptr(modf), ptr(Wf), ptr(bf), ptr(y), R, D, Cout, N, 1e-6, st),
               "ga_final_layer")
    return y, ((xres, modf, Wf) if keep else None)


class _DiTHead(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xres, temb, *params):
        B, N, D = xres.shape
        xf = xres.detach().to(_F32).contiguous().view(B * N, D)
        with torch.cuda.device(xres.device):
            y, saved = _head_forward(xf, temb, params, N, keep=True)
        ctx.save_for_backward(*saved, *params)
        ctx.meta = (xres.shape, xres.dtype, temb.dtype)
        return y.view(B, N, -1)

    @staticmethod
    def backward(ctx, gy):
        if torch.is_grad_enabled():
            raise RuntimeError("dit_grad: double backward (create_graph=True) is not supported")
        with torch.cuda.device(gy.device):
            return _head_backward(ctx, gy)


def _head_backward(ctx, gy):
    xf, modf, Wf, table, W, b = ctx.saved_tensors
    (B, N, D), x_dtype, t_dtype = ctx.meta
    nx, nt, n_tab, n_w, n_b = ctx.needs_input_grad
    R, Cout = B * N, W.shape[0]
    dev = xf.device
    L, st = _lib.lib(), stream(dev)
    P = L.ga_dit_grad_partials(R, N)
    dy = gy.reshape(R, Cout).to(_F32).contiguous()
    dx = torch.empty((R, D), dtype=_F32, device=dev) if nx else None
    pmod = torch.empty((P, 2 * D), dtype=_F32, device=dev) if (nt or n_tab) else None
    pw = torch.empty((P, Cout * D), dtype=_F32, device=dev) if (n_w or n_b) else None
    pb = torch.empty((P, Cout), dtype=_F32, device=dev) if (n_w or n_b) else None
    _lib.check(L.ga_dit_final_layer_bwd(ptr(xf), ptr(modf), ptr(Wf), ptr(dy), ptr(dx), ptr(pmod), ptr(pw), ptr(pb), N,
                                        R, D, Cout, 1e-6, st), "ga_dit_final_layer_bwd")
    grads = [None] * 5
    if nx:
        grads[0] = dx.view(B, N, D).to(x_dtype)
    if nt or n_tab:
        dmod = _reduce(pmod, B, 2 * D)                                   # [B, 2 D]: d shift | d scale
        if nt:
            grads[1] = _reduce(dmod, B, D).to(t_dtype)                   # mod = table + temb: dtemb = dshift + dscale
        if n_tab:
            grads[2] = _reduce(dmod, 1, 2 * D).view(table.shape).to(table.dtype)
    if n_w:
        grads[3] = _reduce(pw, 1, Cout * D).view(W.shape).to(W.dtype)
    if n_b:
        grads[4] = _reduce(pb, 1, Cout)[0].to(b.dtype)
    return tuple(grads)


def _check_model(model, x, timesteps, context):
    from .dit import DiT_I23D_PCD_PixelArt_noclip, ImageCondDiTBlockPixelArtRMSNormClayLRM
    what = type(model).__name__
    if not isinstance(model, DiT_I23D_PCD_PixelArt_noclip):
        raise TypeError("model_forward: %s is not an image-to-3D point DiT" % what)
    if not all(type(b) is ImageCondDiTBlockPixelArtRMSNormClayLRM for b in model.blocks):
        raise NotImplementedError("model_forward: %s has other blocks than ImageCondDiTBlockPixelArtRMSNormClayLRM "
                                  "(the text-to-3D DiT is not trainable here)" % what)
    if model.enable_rope or model.freqs_cis is not None:
        raise NotImplementedError("%s: RoPE is not supported" % what)
    D, heads = model.embed_dim, model.num_heads
    if D % heads or D // heads != 64:
        raise NotImplementedError("%s: head_dim %s is not supported (64 only)" % (what, D / heads))
    Cout, Dc = model.out_channels, model.pooled_vec_embedder[0].weight.shape[0]
    if Cout > 16:
        raise NotImplementedError("%s: out_channels %d > 16 (the final layer's limit)" % (what, Cout))
    if D > 1024 or D % 8 or Dc > 1024 or Dc % 8:
        raise NotImplementedError("%s: hidden size %d or pooled width %d is not a multiple of 8 up to 1024"
                                  % (what, D, Dc))
    if not isinstance(context, dict) or "img_crossattn" not in context or "img_vector" not in context:
        raise ValueError("%s: context must be a dict with img_crossattn and img_vector" % what)
    ctx, vec = context["img_crossattn"], context["img_vector"]
    xyz = context.get("fps-xyz") if model.xyz_cond else None
    if model.xyz_cond and xyz is None:
        raise ValueError("%s: the stage-2 model needs context['fps-xyz']" % what)
    for name, v in (("x", x), ("timesteps", timesteps), ("img_vector", vec), ("fps-xyz", xyz)):
        if v is None and name == "fps-xyz":
            continue
        if not isinstance(v, torch.Tensor):
            raise TypeError("%s: %s must be a tensor" % (what, name))
        if v.dtype not in (torch.float32, torch.bfloat16, torch.float16):
            raise TypeError("%s: %s must be fp32, bf16 or fp16, got %s" % (what, name, v.dtype))
    for name, v in (("timesteps", timesteps), ("context['fps-xyz']", xyz)):
        if v is not None and v.requires_grad:
            raise ValueError("%s: %s is a constant of the model and gets no gradient; pass it detached" % (what, name))
    if x.dim() != 3 or x.shape[2] != model.in_channels or x.shape[0] < 1 or x.shape[1] < 1:
        raise ValueError("%s: x must be [B, N, %d], got %s" % (what, model.in_channels, tuple(x.shape)))
    B, N = x.shape[:2]
    K = model.in_channels + (3 if model.xyz_cond and not model.use_pe_cond else 0)
    if K > 16:
        raise NotImplementedError("%s: the token embedder's %d inputs > 16" % (what, K))
    if timesteps.numel() not in (1, B):
        raise ValueError("%s: timesteps must hold 1 or B = %d values, got %s" % (what, B, tuple(timesteps.shape)))
    if vec.numel() != B * Dc:
        raise ValueError("%s: img_vector must be [%d, %d], got %s" % (what, B, Dc, tuple(vec.shape)))
    if xyz is not None and xyz.numel() != B * N * 3:
        raise ValueError("%s: fps-xyz must be [%d, %d, 3], got %s" % (what, B, N, tuple(xyz.shape)))
    stem, head = stem_parameters(model), head_parameters(model)
    tensors = (x, timesteps, ctx, vec) + ((xyz,) if xyz is not None else ()) + stem + head
    if not all(v.is_cuda for v in tensors):
        raise RuntimeError("%s needs CUDA tensors (there is no CPU fallback)" % what)
    if any(v.device != x.device for v in tensors):
        raise ValueError("%s: inputs and parameters are on different devices" % what)
    return ctx, vec, xyz, stem, head


def model_forward(model, x, timesteps=None, context=None):
    """DiT_I23D_PCD_PixelArt_noclip(_clay_stage2).forward with a backward: x [B, N, in_channels], timesteps [B] (or
    one value), context {img_crossattn [B, M, Dc], img_vector [B, Dc], fps-xyz [B, N, 3] for stage 2}.  Returns y
    [B, N, out_channels] fp32.  Gradients reach x, img_crossattn, img_vector and every parameter the forward reads;
    timesteps and fps-xyz are constants.  functools.partial(model_forward, model) is a model for
    Transport.training_losses.  The model's inference engine (model(...)) is not touched."""
    ctx, vec, xyz, stem, head = _check_model(model, x, timesteps, context)
    B, N = x.shape[:2]
    grad = torch.is_grad_enabled()
    with torch.cuda.device(x.device):
        if grad and any(v.requires_grad for v in (x, vec) + stem):
            xres, t0, temb = _DiTStem.apply(x, vec, timesteps, xyz, *stem)
        else:
            xres, t0, temb, _ = _stem_forward(x, vec, timesteps, xyz, stem, keep=False)
            xres = xres.view(B, N, -1)
        h = xres
        for blk in model.blocks:
            h = block_forward(blk, h, t0, ctx)
        if grad and any(v.requires_grad for v in (h, temb) + head):
            return _DiTHead.apply(h, temb, *head)
        y, _ = _head_forward(h.detach().to(_F32).contiguous().view(B * N, -1), temb, head, N, keep=False)
        return y.view(B, N, -1)
