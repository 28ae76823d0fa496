"""Differentiable `FusedMLP` and `linear` on the library's kernels (include/ga_b200.h Part 13).

xformers' FusedMLP is the second half of every transformer block the reference trains (the image and text DiT blocks,
the VAE decoder's DiT2-B/2 blocks, the decoder's up-sampler transformers and the encoder's SRT layers):

    Linear(D -> m D, no bias) -> + bias, exact GELU -> Linear(m D -> D, no bias) -> + bias

    from gaussiananything_b200.mlp import FusedMLP
    mlp = FusedMLP(dim_model=1024, dropout=0.0, activation="gelu", hidden_layer_multiplier=4).cuda()
    mlp.load_state_dict(sd, strict=True)       # mlp.0.weight, mlp.1.bias, mlp.2.weight, mlp.3.bias
    y = mlp(x)                                 # x [..., 1024]
    y.float().sum().backward()                 # x.grad and every parameter's grad

The forward runs fc1 with an epilogue that keeps the bf16 pre-activation Z next to H = gelu(v); the backward forms
db2, dW2 = dY^T H, dZ = (dY W2) o gelu'(Z) (one fused GEMM), db1, dW1 = dZ^T x and dx = dZ W1, each only when
something needs it.  Under no_grad, or when nothing requires grad, fc1 writes H alone and nothing is saved.
`linear(x, weight, bias)` is the same for one nn.Linear.

Operands are bf16: fp16 and fp32 inputs are rounded on entry, the fp32 parameters are packed to bf16 on every call
(they change every step).  The output and dx come back in x's dtype, parameter gradients in the parameter's dtype.
There is no CPU fallback, no dropout and no other activation: those raise.
"""
import ctypes as C
import importlib
import sys

import torch
from torch import nn

from . import _lib
from ._launch import epilogue, gemm, gemm_config, ptr, stream
from ._lib import EPI_BF16, EPI_F32, EPI_GELU_BF16

__all__ = ["FusedMLP", "fused_mlp", "linear", "install_shims"]

_BF16 = torch.bfloat16


# ---- kernel calls (prepared operands: bf16, contiguous, on one device) -----------------------------------------

def _rows(x, K):
    """x [..., K] as a contiguous bf16 [M, K] matrix (x itself when it already is one)."""
    x2 = x.reshape(-1, K)
    if x2.dtype != _BF16:
        x2 = x2.to(_BF16)
    return x2.contiguous()


def _pack(w):
    """A parameter as the kernels read it: bf16, row-major."""
    return w.detach().to(_BF16).contiguous()


def _bias(b):
    return None if b is None else b.detach().to(torch.float32).contiguous()


def _workspace(nbytes, device):
    return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device)


def _forward_linear(xb, wb, bf, out_dtype):
    """y [M, N] = xb [M, K] wb[N, K]^T + bias, bf16 when out_dtype is bf16, else fp32."""
    M, K = xb.shape
    N = wb.shape[0]
    f32 = out_dtype != _BF16
    y = torch.empty((M, N), dtype=torch.float32 if f32 else _BF16, device=xb.device)
    gemm(xb, wb, M, N, K, epilogue(EPI_F32 if f32 else EPI_BF16, bias=bf if bf is not None else 0, out=y, ld_out=N),
         stream(xb.device))
    return y


def _fc1(xb, w1b, b1f, keep_pre):
    """(H, Z) bf16 [M, hidden]: H = gelu(x W1^T + b1); Z = x W1^T + b1 when keep_pre, else None."""
    M, D = xb.shape
    Hd = w1b.shape[0]
    h = torch.empty((M, Hd), dtype=_BF16, device=xb.device)
    if not keep_pre:
        gemm(xb, w1b, M, Hd, D, epilogue(EPI_GELU_BF16, bias=b1f, out=h, ld_out=Hd), stream(xb.device))
        return h, None
    z = torch.empty_like(h)
    _lib.check(_lib.lib().ga_linear_fc1_gelu_bf16(ptr(xb), ptr(w1b), ptr(b1f), ptr(h), ptr(z), M, Hd, D,
                                                  gemm_config(M, Hd, EPI_GELU_BF16), stream(xb.device)),
               "ga_linear_fc1_gelu_bf16")
    return h, z


def _dgrad(g, wb, z=None, f32=False):
    """g [M, N] wb [N, K] -> [M, K] (fp32 when f32, else bf16); with z: bf16(product o gelu'(z))."""
    M, N = g.shape
    K = wb.shape[1]
    out = torch.empty((M, K), dtype=torch.float32 if f32 else _BF16, device=g.device)
    _lib.check(_lib.lib().ga_linear_dgrad_bf16(ptr(g), ptr(wb), ptr(z), ptr(out), int(f32), M, N, K,
                                               stream(g.device)), "ga_linear_dgrad_bf16")
    return out


def _wgrad(g, x):
    """dW fp32 [N, K] = g [M, N]^T x [M, K]."""
    M, N = g.shape
    K = x.shape[1]
    L = _lib.lib()
    ws_bytes = L.ga_linear_wgrad_workspace_bytes(M, N, K)
    ws = _workspace(ws_bytes, g.device)
    dw = torch.empty((N, K), dtype=torch.float32, device=g.device)
    _lib.check(L.ga_linear_wgrad_bf16(ptr(g), ptr(x), ptr(dw), M, N, K, ptr(ws), ws.numel(), stream(g.device)),
               "ga_linear_wgrad_bf16")
    return dw


def _bgrad(g):
    """db fp32 [N] = column sums of g [M, N]."""
    M, N = g.shape
    L = _lib.lib()
    ws = _workspace(L.ga_linear_bias_grad_workspace_bytes(M, N), g.device)
    db = torch.empty(N, dtype=torch.float32, device=g.device)
    _lib.check(L.ga_linear_bias_grad_bf16(ptr(g), ptr(db), M, N, ptr(ws), ws.numel(), stream(g.device)),
               "ga_linear_bias_grad_bf16")
    return db


def _out(y, shape, dtype):
    y = y.view(shape)
    return y if y.dtype == dtype else y.to(dtype)


# ---- argument checks --------------------------------------------------------------------------------------------

def _check_tensors(what, x, params):
    if not isinstance(x, torch.Tensor):
        raise TypeError("%s: the input must be a tensor" % what)
    if x.dtype not in (torch.bfloat16, torch.float16, torch.float32):
        raise TypeError("%s: the input must be bf16, fp16 or fp32, got %s" % (what, x.dtype))
    if x.dim() < 1 or x.numel() == 0:
        raise ValueError("%s: empty input of shape %s" % (what, tuple(x.shape)))


def _check_device(what, x, params):
    if not x.is_cuda or not all(p.is_cuda for p in params if p is not None):
        raise RuntimeError("%s needs CUDA tensors (there is no CPU fallback)" % what)
    if any(p.device != x.device for p in params if p is not None):
        raise ValueError("%s: the input and the parameters are on different devices" % what)


def _check_width(what, n, name):
    if n < 8 or n % 8:
        raise NotImplementedError("%s: %s = %d is not a multiple of 8 (the kernels' row pitch)" % (what, name, n))


# ---- linear -------------------------------------------------------------------------------------------------------

class _Linear(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias):
        N, K = weight.shape
        xb, wb = _rows(x, K), _pack(weight)
        with torch.cuda.device(x.device):
            y = _forward_linear(xb, wb, _bias(bias), x.dtype)
        ctx.save_for_backward(xb, wb, weight, bias)
        ctx.x_meta = (x.shape, x.dtype)
        return _out(y, x.shape[:-1] + (N,), x.dtype)

    @staticmethod
    def backward(ctx, gy):
        if torch.is_grad_enabled():
            raise RuntimeError("linear: double backward (create_graph=True) is not supported")
        xb, wb, weight, bias = ctx.saved_tensors
        need_x, need_w, need_b = ctx.needs_input_grad
        shape, dtype = ctx.x_meta
        g = _rows(gy, wb.shape[0])
        dx = dw = db = None
        with torch.cuda.device(xb.device):
            if need_x:
                dx = _out(_dgrad(g, wb, f32=dtype != _BF16), shape, dtype)
            if need_w:
                dw = _wgrad(g, xb).to(weight.dtype)
            if need_b:
                db = _bgrad(g).to(bias.dtype)
        return dx, dw, db


def linear(x, weight, bias=None):
    """x [..., K] W^T + bias with a backward, as torch.nn.functional.linear; weight [N, K] (fp32 parameter), N and K
    multiples of 8.  The forward is ga_gemm_bf16_tn; the backward forms dx (dgrad), dW (wgrad) and db as needed."""
    _check_tensors("linear", x, (weight, bias))
    N, K = weight.shape
    if x.shape[-1] != K or (bias is not None and tuple(bias.shape) != (N,)):
        raise ValueError("linear: input %s, weight %s and bias %s do not fit" % (
            tuple(x.shape), tuple(weight.shape), None if bias is None else tuple(bias.shape)))
    _check_width("linear", N, "out_features")
    _check_width("linear", K, "in_features")
    _check_device("linear", x, (weight, bias))
    return _Linear.apply(x, weight, bias)


# ---- FusedMLP -----------------------------------------------------------------------------------------------------

class _FusedMLP(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2):
        D = w1.shape[1]
        xb, w1b, w2b = _rows(x, D), _pack(w1), _pack(w2)
        with torch.cuda.device(x.device):
            h, z = _fc1(xb, w1b, _bias(b1), keep_pre=True)
            y = _forward_linear(h, w2b, _bias(b2), x.dtype)
        # the parameters themselves are saved too, so that changing one in place before backward raises
        ctx.save_for_backward(xb, z, h, w1b, w2b, w1, b1, w2, b2)
        ctx.x_meta = (x.shape, x.dtype)
        return _out(y, x.shape, x.dtype)

    @staticmethod
    def backward(ctx, gy):
        if torch.is_grad_enabled():
            raise RuntimeError("fused_mlp: double backward (create_graph=True) is not supported")
        xb, z, h, w1b, w2b, w1, b1, w2, b2 = ctx.saved_tensors
        need_x, need_w1, need_b1, need_w2, need_b2 = ctx.needs_input_grad
        shape, dtype = ctx.x_meta
        g = _rows(gy, w2b.shape[0])
        dx = dw1 = db1 = dw2 = db2 = None
        with torch.cuda.device(xb.device):
            if need_b2:
                db2 = _bgrad(g).to(b2.dtype)
            if need_w2:
                dw2 = _wgrad(g, h).to(w2.dtype)
            if need_x or need_w1 or need_b1:
                dz = _dgrad(g, w2b, z=z)
                if need_b1:
                    db1 = _bgrad(dz).to(b1.dtype)
                if need_w1:
                    dw1 = _wgrad(dz, xb).to(w1.dtype)
                if need_x:
                    dx = _out(_dgrad(dz, w1b, f32=dtype != _BF16), shape, dtype)
        return dx, dw1, db1, dw2, db2


def fused_mlp(x, w1, b1, w2, b2):
    """gelu(x W1^T + b1) W2^T + b2 with a backward: x [..., D], w1 [hidden, D], b1 [hidden], w2 [D, hidden], b2 [D]
    (D and hidden multiples of 8).  Under no_grad, or when nothing requires grad, the forward saves nothing."""
    _check_tensors("fused_mlp", x, (w1, b1, w2, b2))
    Hd, D = w1.shape
    if (x.shape[-1] != D or tuple(w2.shape) != (D, Hd) or tuple(b1.shape) != (Hd,) or tuple(b2.shape) != (D,)):
        raise ValueError("fused_mlp: input %s does not fit w1 %s, b1 %s, w2 %s, b2 %s" % tuple(
            tuple(t.shape) for t in (x, w1, b1, w2, b2)))
    _check_width("fused_mlp", D, "dim_model")
    _check_width("fused_mlp", Hd, "the hidden width")
    _check_device("fused_mlp", x, (w1, b1, w2, b2))
    if torch.is_grad_enabled() and any(t.requires_grad for t in (x, w1, b1, w2, b2)):
        return _FusedMLP.apply(x, w1, b1, w2, b2)
    xb = _rows(x, D)
    with torch.cuda.device(x.device):
        h, _ = _fc1(xb, _pack(w1), _bias(b1), keep_pre=False)
        y = _forward_linear(h, _pack(w2), _bias(b2), x.dtype)
    return _out(y, x.shape, x.dtype)


class _Bias(nn.Module):
    """Holds one bias where xformers' FusedDropoutBias keeps it (so the state-dict key is mlp.<i>.bias)."""

    def __init__(self, n):
        super().__init__()
        self.bias = nn.Parameter(torch.zeros(n))


def _is_gelu(activation):
    return str(getattr(activation, "value", activation)).lower() == "gelu"


class FusedMLP(nn.Module):
    """xformers.components.feedforward.fused_mlp.FusedMLP on the library's kernels, with a backward.  The parameters
    are fp32 under xformers' keys (mlp.0.weight [hidden, D], mlp.1.bias [hidden], mlp.2.weight [D, hidden],
    mlp.3.bias [D]); weights take nn.Linear's initialisation and biases start at zero.  Dropout, activations other
    than GeLU, bias=False and widths that are not multiples of 8 raise NotImplementedError."""

    def __init__(self, dim_model, dropout, activation, hidden_layer_multiplier, bias=True, *args, **kwargs):
        super().__init__()
        if dropout > 0:
            raise NotImplementedError("FusedMLP: dropout > 0 is not supported")
        if not _is_gelu(activation):
            raise NotImplementedError("FusedMLP: activation %r is not supported (GeLU only)" % (activation,))
        if not bias:
            raise NotImplementedError("FusedMLP: bias=False is not supported")
        dim_mlp = int(hidden_layer_multiplier * dim_model)
        _check_width("FusedMLP", dim_model, "dim_model")
        _check_width("FusedMLP", dim_mlp, "the hidden width")
        self.mlp = nn.Sequential(nn.Linear(dim_model, dim_mlp, bias=False), _Bias(dim_mlp),
                                 nn.Linear(dim_mlp, dim_model, bias=False), _Bias(dim_model))

    def forward(self, inputs):
        return fused_mlp(inputs, self.mlp[0].weight, self.mlp[1].bias, self.mlp[2].weight, self.mlp[3].bias)


def install_shims():
    """Opt-in: makes xformers.components.feedforward.fused_mlp.FusedMLP this class.  The reference looks the class up
    through that module when it builds a network, so networks built afterwards use it.  Returns False, and changes
    nothing, when that module cannot be imported.  gaussiananything_b200.install_shims() does not call this."""
    name = "xformers.components.feedforward.fused_mlp"
    fm = sys.modules.get(name)
    if fm is None:
        try:
            fm = importlib.import_module(name)
        except Exception:
            return False
    fm.FusedMLP = FusedMLP
    return True
