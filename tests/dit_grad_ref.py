"""fp64 references of the trainable DiT block (include/ga_b200.h Part 14, gaussiananything_b200/dit_grad.py) for the
dit_grad tests: torch only, no library import.

block(P, x, t, ctx, heads, dy) is oracle/dit_oracle.block_forward, which tests/test_oracle_dit.py pins to the
reference's own code, run in float64 under torch autograd: {y, dx, dt, dctx, and one entry per parameter name}.
With emulate=True the same forward is restated with bf16 rounding where the kernels round:
  forward   the GEMM weights; the context; h0, h1, h2 (the norm outputs); the to_q, kv and qkv GEMM outputs; the
            normalised q and k; the attention's P (before P V) and output o; fc1's Z (gelu' is evaluated there) and
            H = gelu(v);
  backward  the gradients of a1, a2, a3 (da = bf16(gate dy), bf16(dx1)), of o (the dgrad's bf16 output), of the
            normalised q, k and of v (the attention's bf16 dq, dk, dv), of the pre-norm q, k and the qkv / kv GEMM
            outputs (the q/k-norm backward's bf16 output), of fc1's pre-activation (dZ = bf16(dH gelu'(Z))) and the
            attention's dS (before dS k and dS^T q).
Everything else (norms, residuals, gates, modulation, the products and all sums) stays fp64 where the kernels use
fp32.  The GPU tests hold each result's L2 distance from fp64 to 1.5 times the emulation's, plus a floor of 2^-16 of
the result's norm.
"""
import math

import torch
import torch.nn.functional as F

PARAMS = ("scale_shift_table", "prenorm_ca_dino.weight", "norm1.weight", "norm2.weight",
          "cross_attn_dino.to_q.weight", "cross_attn_dino.to_k.weight", "cross_attn_dino.to_v.weight",
          "cross_attn_dino.q_norm.weight", "cross_attn_dino.k_norm.weight",
          "cross_attn_dino.to_out.0.weight", "cross_attn_dino.to_out.0.bias",
          "attn.qkv.weight", "attn.qkv.bias", "attn.q_norm.weight", "attn.k_norm.weight",
          "attn.proj.weight", "attn.proj.bias",
          "mlp.mlp.0.weight", "mlp.mlp.1.bias", "mlp.mlp.2.weight", "mlp.mlp.3.bias")
GEMM_WEIGHTS = {k for k in PARAMS if k.endswith("weight") and ("to_" in k or "qkv" in k or "proj" in k
                                                               or "mlp.mlp" in k)}
EPS = 1e-5


def bf16(t):
    return t.to(torch.bfloat16).to(t.dtype)


class _RoundGrad(torch.autograd.Function):
    @staticmethod
    def forward(ctx, t):
        return t.view_as(t)

    @staticmethod
    def backward(ctx, g):
        return bf16(g)


def _rf(t):
    """bf16(t) in the forward, the gradient passed straight through"""
    return t + (bf16(t) - t).detach()


def _rr(t):
    return _RoundGrad.apply(_rf(t))


def _gelu(v):
    return 0.5 * v * (1.0 + torch.erf(v / math.sqrt(2.0)))


def _gelu_grad(z):
    return 0.5 * (1.0 + torch.erf(z / math.sqrt(2.0))) + z * torch.exp(-0.5 * z * z) / math.sqrt(2.0 * math.pi)


class _GeluEmu(torch.autograd.Function):
    """H = bf16(gelu(v)); dZ = bf16(dH gelu'(bf16(v)))"""
    @staticmethod
    def forward(ctx, v):
        ctx.save_for_backward(bf16(v))
        return bf16(_gelu(v))

    @staticmethod
    def backward(ctx, g):
        z, = ctx.saved_tensors
        return bf16(g * _gelu_grad(z))


def _rms(x, w):
    return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + EPS) * w


def _attention(q, k, v, rg, rf):
    """q [B, H, Nq, 64], k, v [B, H, Nk, 64]: softmax(q k^T / 8) v"""
    s = rg(q @ k.transpose(-1, -2)) / 8.0
    return rf(torch.softmax(s, -1)) @ v


def _block_emu(P, x, t, ctx, H, rounding=True):
    """The block restated with the kernels' bf16 roundings (none when rounding is False: then it is the oracle's
    block_forward in another form, which tests/test_dit_grad_cpu.py checks)."""
    ident = lambda u: u
    rf, rr, rg = (_rf, _rr, _RoundGrad.apply) if rounding else (ident, ident, ident)
    gelu = _GeluEmu.apply if rounding else _gelu
    B, N, D = x.shape
    M = ctx.shape[1]
    W = {k: (rf(v) if k in GEMM_WEIGHTS else v) for k, v in P.items()}
    mod = P["scale_shift_table"][None] + t.reshape(B, 6, D)
    s_msa, c_msa, g_msa, s_mlp, c_mlp, g_mlp = (mod[:, j:j + 1] for j in range(6))
    heads = lambda u, n: u.reshape(B, n, H, 64).transpose(1, 2)
    merge = lambda u: u.transpose(1, 2).reshape(B, -1, D)
    # cross-attention
    h0 = rf(_rms(x, P["prenorm_ca_dino.weight"]))
    c = rf(ctx)
    q = rr(F.linear(h0, W["cross_attn_dino.to_q.weight"]))
    k = rr(F.linear(c, W["cross_attn_dino.to_k.weight"]))
    v = rr(F.linear(c, W["cross_attn_dino.to_v.weight"]))
    qn = rr(_rms(heads(q, N), P["cross_attn_dino.q_norm.weight"]))
    kn = rr(_rms(heads(k, M), P["cross_attn_dino.k_norm.weight"]))
    o = rr(merge(_attention(qn, kn, heads(v, M), rg, rf)))
    x1 = x + rg(F.linear(o, W["cross_attn_dino.to_out.0.weight"], P["cross_attn_dino.to_out.0.bias"]))
    # gated self-attention
    h1 = rf(_rms(x1, P["norm1.weight"]) * (1 + c_msa) + s_msa)
    qkv = rr(F.linear(h1, W["attn.qkv.weight"], P["attn.qkv.bias"]))
    q, k, v = qkv.split(D, -1)
    qn = rr(_rms(heads(q, N), P["attn.q_norm.weight"]))
    kn = rr(_rms(heads(k, N), P["attn.k_norm.weight"]))
    o = rr(merge(_attention(qn, kn, heads(v, N), rg, rf)))
    x2 = x1 + g_msa * rg(F.linear(o, W["attn.proj.weight"], P["attn.proj.bias"]))
    # gated FFN
    h2 = rf(_rms(x2, P["norm2.weight"]) * (1 + c_mlp) + s_mlp)
    hid = gelu(F.linear(h2, W["mlp.mlp.0.weight"]) + P["mlp.mlp.1.bias"])
    return x2 + g_mlp * rg(F.linear(hid, W["mlp.mlp.2.weight"]) + P["mlp.mlp.3.bias"])


def block(P, x, t, ctx, heads, dy, emulate=False, restated=False):
    """{name: fp64 tensor}: y and the gradients of x, t, ctx and every parameter (by its state-dict name) for the
    output gradient dy, on the device the tensors are on.  restated: the emulation's code without its roundings."""
    from oracle import dit_oracle
    leaves = {k: P[k].detach().double().clone().requires_grad_(True) for k in PARAMS}
    xs = [v.detach().double().clone().requires_grad_(True) for v in (x, t, ctx)]
    with torch.enable_grad():
        if emulate or restated:
            y = _block_emu(leaves, *xs, heads, rounding=emulate)
        else:
            y = dit_oracle.block_forward(leaves, "", xs[0], xs[1], xs[2], heads)
        y.backward(dy.double())
    out = dict(y=y.detach(), dx=xs[0].grad, dt=xs[1].grad, dctx=xs[2].grad)
    out.update({k: v.grad for k, v in leaves.items()})
    return out


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-300))
