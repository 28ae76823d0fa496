"""Differentiable `memory_efficient_attention` on the library's kernels (include/ga_b200.h Part 12).

A drop-in for `xformers.ops.memory_efficient_attention(query, key, value, attn_bias=None, p=0.0, scale=None, op=None)`,
the one function every transformer the reference trains sends its attention through (INTEGRATION.md section 3k):

    from gaussiananything_b200.attention import memory_efficient_attention
    out = memory_efficient_attention(q, k, v)            # q [B, Mq, H, K], k [B, Mk, H, K], v [B, Mk, H, Kv]
    out.float().sum().backward()                          # q.grad, k.grad, v.grad

Inputs are BMHK ([batch, tokens, heads, d], any strides with a contiguous d: the `unbind` views of a packed qkv) or
BMK ([batch, tokens, d]); the output has the query's layout, the value's last dimension and the query's dtype.  bf16
is computed natively; fp16 and fp32 inputs are rounded to bf16 on entry, as the library's other networks do, and
their gradients come back in their own dtype.  Head dimensions 32 and 64.  The kernels read the tensors where they
lie; only a tensor whose strides they cannot address (not a multiple of 8 elements, or a strided last dimension) is
copied to a contiguous one first.

There is no CPU fallback, no attention bias and no dropout: those raise.
"""
import ctypes as C
import sys

import torch

from . import _lib
from ._launch import ptr, stream

__all__ = ["memory_efficient_attention", "install_shims"]

_BF16 = torch.bfloat16


def _addressable(x):
    """True when the kernels can read x [B, N, H, d] in place: bf16, d contiguous, 16-byte base, strides % 8 == 0."""
    if x.dtype != _BF16 or x.stride(-1) != 1 or x.data_ptr() % 16 != 0:
        return False
    return all(s % 8 == 0 for n, s in zip(x.shape[:-1], x.stride()[:-1]) if n > 1)


def _prepare(x):
    """x as a bf16 [B, N, H, d] tensor the kernels can address: x itself when it can be, else a contiguous copy."""
    if x.dtype != _BF16:
        x = x.to(_BF16)
    return x if _addressable(x) else x.contiguous()


def _strides(x):
    """(batch, token, head) element strides of a 4-D tensor; a size-1 dimension's stride is irrelevant: 0."""
    return [s if n > 1 else 0 for n, s in zip(x.shape[:3], x.stride()[:3])]


def _stride_table(tensors):
    vals = []
    for t in tensors:
        vals += _strides(t) if t is not None else [0, 0, 0]
    return (C.c_int64 * 24)(*vals)


def _check_args(query, key, value, attn_bias, p):
    if attn_bias is not None:
        raise NotImplementedError("memory_efficient_attention: attn_bias is not supported (only attn_bias=None)")
    if p > 0.0:
        raise NotImplementedError("memory_efficient_attention: dropout (p > 0) is not supported")
    for name, t in (("query", query), ("key", key), ("value", value)):
        if not isinstance(t, torch.Tensor):
            raise TypeError("memory_efficient_attention: %s must be a tensor" % name)
        if t.dim() not in (3, 4):
            raise ValueError("memory_efficient_attention: %s must be BMHK (4-D) or BMK (3-D), got shape %s"
                             % (name, tuple(t.shape)))
        if t.shape[-1] not in (32, 64):
            raise NotImplementedError("memory_efficient_attention: head dimension %d of %s is not supported "
                                      "(32 or 64)" % (t.shape[-1], name))
        if t.dtype not in (torch.bfloat16, torch.float16, torch.float32):
            raise TypeError("memory_efficient_attention: %s must be bf16, fp16 or fp32, got %s" % (name, t.dtype))
    if not (query.dim() == key.dim() == value.dim()):
        raise ValueError("memory_efficient_attention: query, key and value must all be BMHK or all BMK")
    if query.shape[-1] != key.shape[-1]:
        raise ValueError("memory_efficient_attention: query and key head dimensions differ: %d, %d"
                         % (query.shape[-1], key.shape[-1]))
    if key.shape[:-1] != value.shape[:-1]:
        raise ValueError("memory_efficient_attention: key %s and value %s disagree outside the last dimension"
                         % (tuple(key.shape), tuple(value.shape)))
    if query.shape[0] != key.shape[0] or (query.dim() == 4 and query.shape[2] != key.shape[2]):
        raise ValueError("memory_efficient_attention: query %s and key %s disagree in batch or heads"
                         % (tuple(query.shape), tuple(key.shape)))
    if query.shape[1] < 1 or key.shape[1] < 1 or query.shape[0] < 1 or (query.dim() == 4 and query.shape[2] < 1):
        raise ValueError("memory_efficient_attention: empty query or key")
    if not (query.is_cuda and key.is_cuda and value.is_cuda):
        raise RuntimeError("memory_efficient_attention needs CUDA tensors (there is no CPU fallback)")
    if not (query.device == key.device == value.device):
        raise ValueError("memory_efficient_attention: query, key and value are on different devices")


def _non_overlapping(shape, stride):
    """True when no two indices of a tensor with this shape and these strides share an element (an `expand`ed
    dimension, stride 0 with size > 1, does)."""
    extent = 1
    for s, n in sorted((s, n) for n, s in zip(shape, stride) if n > 1):
        if s < extent:
            return False
        extent = s * n
    return True


def _grad_buffer(x):
    """An uninitialised bf16 gradient for the prepared input x: x's own strides when no two of its indices share an
    element (the kernels then write it in the layout the input has), else contiguous.  Every (batch, head) CTA writes
    its own rows, so an overlapping layout (an expanded input) would make them overwrite each other."""
    if _non_overlapping(x.shape, x.stride()):
        return torch.empty_strided(x.shape, x.stride(), dtype=_BF16, device=x.device)
    return torch.empty(x.shape, dtype=_BF16, device=x.device)


def _grad_like(buf, orig):
    """The gradient in buf (bf16, [B, N, H, d]) as a tensor with the input's (shape, dtype) and its strides when they
    do not overlap (an expanded input gets a contiguous gradient; autograd sums it over the expanded dimension)."""
    shape, stride, dtype = orig
    if buf.dim() != len(shape):
        buf = buf.squeeze(2)
    if buf.dtype == dtype and (buf.stride() == stride or not _non_overlapping(shape, stride)):
        return buf
    if _non_overlapping(shape, stride):
        out = torch.empty_strided(shape, stride, dtype=dtype, device=buf.device)
    else:
        out = torch.empty(shape, dtype=dtype, device=buf.device)
    return out.copy_(buf)


def _forward(qp, kp, vp, scale):
    """(o bf16 [B, Nq, H, Dv], lse fp32 [B * H, Nq]) of prepared [B, N, H, d] tensors."""
    B, Nq, H, D = qp.shape
    Nk, Dv = kp.shape[1], vp.shape[3]
    dev = qp.device
    o = torch.empty((B, Nq, H, Dv), dtype=_BF16, device=dev)
    lse = torch.empty((B * H, Nq), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().ga_attention_fwd_lse_bf16(ptr(qp), ptr(kp), ptr(vp), ptr(o), ptr(lse), B, H, Nq, Nk, D,
                                                        Dv, _stride_table((qp, kp, vp, o)), float(scale), stream(dev)),
                   "ga_attention_fwd_lse_bf16")
    return o, lse


def _backward(qp, kp, vp, o, lse, g, dq, dk, dv, scale):
    """Writes the gradients dq, dk, dv (each may be None) of prepared [B, N, H, d] tensors, given _forward's o and lse
    and the output gradient g, into those [B, N, H, d] buffers."""
    B, Nq, H, D = qp.shape
    Nk, Dv = kp.shape[1], vp.shape[3]
    dev = qp.device
    delta = torch.empty((B * H, Nq), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().ga_attention_bwd_bf16(ptr(qp), ptr(kp), ptr(vp), ptr(o), ptr(lse), ptr(g), ptr(delta),
                                                    ptr(dq), ptr(dk), ptr(dv), B, H, Nq, Nk, D, Dv,
                                                    _stride_table((qp, kp, vp, o, g, dq, dk, dv)), float(scale),
                                                    stream(dev)),
                   "ga_attention_bwd_bf16")


class _MemEffAttention(torch.autograd.Function):
    @staticmethod
    def forward(ctx, query, key, value, scale):
        bmk = query.dim() == 3
        q4, k4, v4 = (t.unsqueeze(2) if bmk else t for t in (query, key, value))
        qp, kp, vp = _prepare(q4), _prepare(k4), _prepare(v4)
        B, Nq, _, Dv = qp.shape[0], qp.shape[1], qp.shape[2], vp.shape[3]
        o, lse = _forward(qp, kp, vp, scale)
        ctx.save_for_backward(qp, kp, vp, o, lse)
        ctx.scale = float(scale)
        ctx.orig = [(t.shape, t.stride(), t.dtype) for t in (query, key, value)]
        out = o.view(B, Nq, Dv) if bmk else o
        return out if query.dtype == _BF16 else out.to(query.dtype)

    @staticmethod
    def backward(ctx, grad_out):
        if torch.is_grad_enabled():
            raise RuntimeError("memory_efficient_attention: double backward (create_graph=True) is not supported")
        qp, kp, vp, o, lse = ctx.saved_tensors
        need_q, need_k, need_v = ctx.needs_input_grad[:3]
        g = grad_out.unsqueeze(2) if grad_out.dim() == 3 else grad_out
        g = _prepare(g)
        # the gradients are written with the strides of the tensors the kernels read (the inputs' own when bf16)
        dq = _grad_buffer(qp) if need_q else None
        dk = _grad_buffer(kp) if need_k else None
        dv = _grad_buffer(vp) if need_v else None
        _backward(qp, kp, vp, o, lse, g, dq, dk, dv, ctx.scale)
        oq, ok, ov = ctx.orig
        return (_grad_like(dq, oq) if need_q else None, _grad_like(dk, ok) if need_k else None,
                _grad_like(dv, ov) if need_v else None, None)


def memory_efficient_attention(query, key, value, attn_bias=None, p=0.0, scale=None, *, op=None):
    """softmax(query key^T * scale) value, as xformers.ops.memory_efficient_attention computes it, with a backward.
    `scale` defaults to query.shape[-1] ** -0.5; `op` is accepted and ignored."""
    _check_args(query, key, value, attn_bias, p)
    if scale is None:
        scale = query.shape[-1] ** -0.5
    return _MemEffAttention.apply(query, key, value, float(scale))


def install_shims():
    """Opt-in: makes xformers.ops.memory_efficient_attention (and the name vit.vision_transformer bound at import, when
    that module is loaded) this function.  Leaves everything alone when xformers.ops cannot be imported.  Returns True
    when it swapped.  gaussiananything_b200.install_shims() does not call this (INTEGRATION.md section 3k)."""
    xops = sys.modules.get("xformers.ops")
    if xops is None:
        try:
            import xformers.ops as xops
        except Exception:
            return False
    xops.memory_efficient_attention = memory_efficient_attention
    vt = sys.modules.get("vit.vision_transformer")
    if vt is not None and hasattr(vt, "memory_efficient_attention"):
        vt.memory_efficient_attention = memory_efficient_attention
    return True
