"""fp64 attention forward and backward for the memory_efficient_attention tests (torch only, no library import), a
bf16-emulating variant, and per-element bounds for O and lse.

attention_fwd / attention_bwd take [BH, N, d] tensors that hold bf16 values (the kernels' inputs, d = 32 or 64) and
work in fp64.  With emulate=True they round where the tiled kernels (include/ga_b200.h Part 12) round:
  forward   P = exp(S - max) rounded to bf16 before P V (the row sum l uses the unrounded P), O rounded to bf16;
  backward  P rounded to bf16 before P^T dO, dS rounded to bf16 before dS^T q and dS k, dq, dk, dv rounded to bf16;
            Delta = rowsum(dO o O) from the bf16 O.
Inputs and dO are bf16 already, so both variants see the same operands.  The GPU tests hold each gradient's L2
distance from fp64 to 1.5 times the emulation's, plus grad_floors (2^-16 of a norm bound of the gradient).  The
emulation's relative distances from fp64,  measured on the CPU with randn inputs (q, k scaled by 1.2, scale 1/8):
  [BH 2, Nq 129, Nk 127, d 64]   O 2.0e-3  dq 2.6e-3  dk 2.5e-3  dv 2.3e-3
  [BH 4, Nq 768, Nk 768, d 64]   O 2.1e-3  dq 2.4e-3  dk 2.4e-3  dv 2.4e-3
  [BH 8, Nq 9,   Nk 9,   d 64]   O 1.9e-3  dq 2.7e-3  dk 2.6e-3  dv 2.5e-3
  [BH 4, Nq 300, Nk 77,  d 32]   O 2.1e-3  dq 2.5e-3  dk 2.4e-3  dv 2.4e-3
The fp64 variant matches torch autograd through softmax(q k^T s) v in fp64 to 1e-15 on the same shapes.
The short path (Nq, Nk <= 16) does not round P or dS, so it sits closer to fp64 than the emulation.

O and lse are also checked element by element (tests/tc_ref.py's attention bound for O; for lse the fp32 score error
ACC |scale| max_j sum_c |q_c k_jc| plus 2^-20 |lse|).

The large shapes run on the GPU in fp64, chunked over query rows; dk and dv add the chunks in order.
"""
import torch

from tests import tc_ref


def bf16(x):
    return x.to(torch.bfloat16).to(torch.float64)


def attention_fwd(q, k, v, scale, emulate=False, chunk=1024):
    """(O, lse, O_tol, lse_tol), fp64: O [BH, Nq, dv], lse [BH, Nq]."""
    q, k, v = q.double(), k.double(), v.double()
    BH, Nq, _ = q.shape
    O = torch.empty(BH, Nq, v.shape[-1], dtype=torch.float64, device=q.device)
    lse = torch.empty(BH, Nq, dtype=torch.float64, device=q.device)
    To = torch.empty_like(O)
    Tl = torch.empty_like(lse)
    vmax = v.abs().amax(dim=(1, 2), keepdim=True)
    for c0 in range(0, Nq, chunk):
        qc = q[:, c0:c0 + chunk]
        s = torch.einsum("bqd,bkd->bqk", qc, k) * scale
        m = s.amax(-1, keepdim=True)
        e = torch.exp(s - m)
        l = e.sum(-1, keepdim=True)
        lse[:, c0:c0 + chunk] = (m + torch.log(l)).squeeze(-1)
        o = torch.einsum("bqk,bkd->bqd", bf16(e) if emulate else e, v) / l
        O[:, c0:c0 + chunk] = bf16(o) if emulate else o
        p = e / l
        To[:, c0:c0 + chunk] = (tc_ref.ATTN_P * torch.einsum("bqk,bkd->bqd", p, v.abs()) + tc_ref.BF16 * o.abs()
                                + tc_ref.ATTN_FLOOR * vmax)
        sabs = torch.einsum("bqd,bkd->bqk", qc.abs(), k.abs()).amax(-1) * abs(scale)
        Tl[:, c0:c0 + chunk] = tc_ref.ACC * sabs + 2.0 ** -20 * lse[:, c0:c0 + chunk].abs() + 1e-6
    return O, lse, To, Tl


def attention_bwd(q, k, v, o, lse, do, scale, emulate=False, chunk=1024):
    """(dq, dk, dv) fp64 from the forward's O and lse (fp64 tensors of attention_fwd with the same emulate)."""
    q, k, v, o, do = q.double(), k.double(), v.double(), o.double(), do.double()
    rnd = bf16 if emulate else (lambda x: x)
    BH, Nq, _ = q.shape
    dq = torch.empty_like(q)
    dk = torch.zeros_like(k)
    dv = torch.zeros_like(v)
    delta = (do * o).sum(-1)
    for c0 in range(0, Nq, chunk):
        sl = slice(c0, c0 + chunk)
        s = torch.einsum("bqd,bkd->bqk", q[:, sl], k) * scale
        p = torch.exp(s - lse[:, sl, None])
        dp = torch.einsum("bqd,bkd->bqk", do[:, sl], v)
        ds = rnd(p * (dp - delta[:, sl, None]))
        dv += torch.einsum("bqk,bqd->bkd", rnd(p), do[:, sl])
        dk += torch.einsum("bqk,bqd->bkd", ds, q[:, sl])
        dq[:, sl] = torch.einsum("bqk,bkd->bqd", ds, k) * scale
    dk *= scale
    return rnd(dq), rnd(dk), rnd(dv)


def grad_floors(q, k, v, do, scale):
    """Absolute L2 floors of (dq, dk, dv): 2^-16 times a norm bound of each gradient, so a gradient that is exactly
    zero in fp64 (one key: softmax is 1 and dS = 0) is compared against fp32 cancellation, not against zero."""
    q, k, v, do = q.double(), k.double(), v.double(), do.double()
    rn = lambda t: float(t.norm(dim=-1).max())
    g = float(do.norm()) * rn(v)
    return 2.0 ** -16 * abs(scale) * g * rn(k), 2.0 ** -16 * abs(scale) * g * rn(q), 2.0 ** -16 * float(do.norm())


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def inputs(BH, Nq, Nk, d, gen, dv=None, qk_scale=1.2, device="cpu"):
    """bf16 q, k, v, dO [BH, N, d] from randn (q, k scaled by qk_scale)."""
    dv = d if dv is None else dv
    r = lambda *s: torch.randn(*s, generator=gen)
    q = (r(BH, Nq, d) * qk_scale).to(torch.bfloat16)
    k = (r(BH, Nk, d) * qk_scale).to(torch.bfloat16)
    v = r(BH, Nk, dv).to(torch.bfloat16)
    do = r(BH, Nq, dv).to(torch.bfloat16)
    return tuple(t.to(device) for t in (q, k, v, do))
