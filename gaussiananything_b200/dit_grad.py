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
from ._launch import ptr, stream
from .attention import _stride_table
from .mlp import _bgrad, _dgrad, _fc1, _forward_linear, _pack, _wgrad

__all__ = ["block_forward"]

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


def _attention(q, k, v, B, H, N, M):
    o = torch.empty((B, N, H, 64), dtype=_BF16, device=q.device)
    lse = torch.empty((B * H, N), dtype=_F32, device=q.device)
    _lib.check(_lib.lib().ga_attention_fwd_lse_bf16(ptr(q), ptr(k), ptr(v), ptr(o), ptr(lse), B, H, N, M, 64, 64,
                                                    _stride_table((q, k, v, o)), _SCALE, stream(q.device)),
               "ga_attention_fwd_lse_bf16")
    return o, lse


def _attention_bwd(q, k, v, o, lse, g, dq, dk, dv, B, H, N, M):
    delta = torch.empty((B * H, N), dtype=_F32, device=q.device)
    _lib.check(_lib.lib().ga_attention_bwd_bf16(ptr(q), ptr(k), ptr(v), ptr(o), ptr(lse), ptr(g), ptr(delta),
                                                ptr(dq), ptr(dk), ptr(dv), B, H, N, M, 64, 64,
                                                _stride_table((q, k, v, o, g, dq, dk, dv)), _SCALE, stream(q.device)),
               "ga_attention_bwd_bf16")


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
    o_ca, lse_ca = _attention(qcn.view(B, N, H, 64), kcn.view(B, M, H, 64), _heads(kv, B, M, 2, 1), B, H, N, M)
    a1 = _forward_linear(o_ca.view(R, D), wo, o_bf, _F32)
    x1, h1 = torch.empty_like(xf), torch.empty_like(h0)
    _gate_residual(xf, a1, None, x1, n1_f, ch(0), ch(1), h1, N, D)
    # gated self-attention
    qkv = _forward_linear(h1, wqkv, qkv_bf, _BF16)                      # [B N, 3 D]: q | k | v
    qkn = _qk_norm(qkv, 3 * D, qn_f, kn_f, R, H, 2)
    o_sa, lse_sa = _attention(_heads(qkn, B, N, 2, 0), _heads(qkn, B, N, 2, 1), _heads(qkv, B, N, 3, 2), B, H, N, N)
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
                           do, _heads(dqkv, B, N, 3, 0), _heads(dqkv, B, N, 3, 1), _heads(dqkv, B, N, 3, 2),
                           B, H, N, N)
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
                           _heads(dkv, B, M, 2, 1) if kv_side else None, B, H, N, M)
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
