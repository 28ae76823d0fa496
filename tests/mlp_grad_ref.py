"""fp64 FusedMLP forward and backward for the mlp tests (torch only, no library import), a bf16-emulating variant,
and per-element bounds of the linear-gradient kernels (include/ga_b200.h Part 13).

mlp(x, w1, b1, w2, b2, dy) works in fp64 on whatever values it is given.  With emulate=True it rounds where the
kernels round: the GEMM operands x, W1, W2 and dY to bf16, Z = bf16(v) and H = bf16(gelu(v)) with v = x W1^T + b1,
dZ = bf16((dY W2) o gelu'(Z)) evaluated at the bf16 Z, and db1 from the bf16 dZ; everything else (the products, dW,
db, y and dx) stays fp64, where the kernels accumulate in fp32.  The fp64 variant rounds nothing.
The GPU tests hold each result's L2 distance from fp64 to 1.5 times the emulation's, plus a floor of 2^-16 of a norm
bound of the result (`floor`).  The emulation's relative distances from fp64, measured on the CPU with x ~ randn,
nn.Linear-initialised weights, biases ~ 0.1 randn and dY ~ randn (fp64 values, so the rounding of x and dY counts):
  [M 300, D 64, hidden 256]    H 2.8e-3  Z 2.8e-3  y 2.8e-3  dZ 3.1e-3  dx 3.5e-3  dW1 3.6e-3  dW2 3.2e-3  db1 3.0e-3
                               db2 1.7e-3
  [M 768, D 256, hidden 1024]  H 2.8e-3  Z 2.8e-3  y 2.9e-3  dZ 3.1e-3  dx 3.5e-3  dW1 3.6e-3  dW2 3.3e-3  db1 3.1e-3
                               db2 1.7e-3
Where dY already holds bf16 values (the kernel tests), the emulation's db2 is exact and the floor alone bounds it.
"""
import math

import torch

# per-element bounds (see tests/tc_ref.py for ACC, BF16, F32)
ACC = 2.0 ** -12
BF16 = 2.0 ** -8
F32 = 2.0 ** -23
U32 = 2.0 ** -24
GELU_D = 1.13              # max |gelu'|
GELU_GRAD_ARITH = 2.0 ** -18   # fp32 erff / expf evaluation of gelu'(z), absolute


def bf16(t):
    return t.to(torch.bfloat16).to(t.dtype)


def gelu(v):
    return 0.5 * v * (1.0 + torch.erf(v / math.sqrt(2.0)))


def gelu_grad(z):
    return 0.5 * (1.0 + torch.erf(z / math.sqrt(2.0))) + z * torch.exp(-0.5 * z * z) / math.sqrt(2.0 * math.pi)


def mlp(x, w1, b1, w2, b2, dy, emulate=False):
    """{name: fp64 tensor} of the forward (v, Z, H, y) and backward (dZ, dx, dW1, db1, dW2, db2) of
    gelu(x W1^T + b1) W2^T + b2 for x [M, D] and the output gradient dy [M, D]."""
    r = bf16 if emulate else (lambda t: t)
    x, w1, b1, w2, b2, dy = (t.double() for t in (x, w1, b1, w2, b2, dy))
    xb, w1b, w2b, g = r(x), r(w1), r(w2), r(dy)
    v = xb @ w1b.T + b1
    z = r(v)
    h = r(gelu(v))
    y = h @ w2b.T + b2
    dh = g @ w2b
    dz = r(dh * gelu_grad(z))
    return dict(v=v, Z=z, H=h, y=y, dH=dh, dZ=dz, dx=dz @ w1b, dW1=dz.T @ xb, db1=dz.sum(0), dW2=g.T @ h,
                db2=g.sum(0))


def mlp_autograd(x, w1, b1, w2, b2, dy):
    """The same in fp64 through torch autograd (nn.functional, exact GELU): {y, dx, dW1, db1, dW2, db2}."""
    ts = [t.double().clone().requires_grad_(True) for t in (x, w1, b1, w2, b2)]
    x_, w1_, b1_, w2_, b2_ = ts
    y = torch.nn.functional.linear(torch.nn.functional.gelu(torch.nn.functional.linear(x_, w1_, b1_)), w2_, b2_)
    y.backward(dy.double())
    return dict(y=y.detach(), dx=x_.grad, dW1=w1_.grad, db1=b1_.grad, dW2=w2_.grad, db2=b2_.grad)


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-300))


def floor(*factors):
    """2^-16 of a norm bound of a product of the given tensors' norms (an absolute slack for the L2 checks)."""
    n = 1.0
    for f in factors:
        n *= float(f.double().norm())
    return 2.0 ** -16 * n


# ---- per-element bounds of single kernels (operands hold exact bf16 values) -------------------------------------

def product(A, B):
    """A [M, C] B [C, N] in fp64 and S = |A| |B| (the magnitude of the summed terms)."""
    a, b = A.double(), B.double()
    return a @ b, a.abs() @ b.abs()


def fc1_bounds(x, w1, b1):
    """(v, Z tol, H ref, H tol) of ga_linear_fc1_gelu_bf16 on bf16 x [M, D], w1 [hidden, D], fp32 b1."""
    v, S = product(x, w1.T)
    v = v + b1.double()
    S = S + b1.double().abs()
    h = gelu(v)
    return (v, ACC * S + (BF16 + F32) * v.abs(), h,
            GELU_D * ACC * S + 2.0 ** -17 * v.abs() + (BF16 + F32) * h.abs())


def dgrad_bounds(g, w, z=None, out_bf16=True):
    """(ref, tol) of ga_linear_dgrad_bf16: g [M, N] w [N, K] (bf16 values), times gelu'(z) when z is given."""
    p, S = product(g, w)
    rnd = BF16 + F32 if out_bf16 else F32
    if z is None:
        return p, ACC * S + rnd * p.abs()
    gz = gelu_grad(z.double())
    ref = p * gz
    return ref, ACC * S * gz.abs() + GELU_GRAD_ARITH * p.abs() + rnd * ref.abs()


def wgrad_bounds(g, x):
    """(ref, tol) of ga_linear_wgrad_bf16: dW [N, K] = g [M, N]^T x [M, K].  The fp32 sum runs over M terms (in at
    most 32 split partials), so the accumulation bound is max(ACC, (M + 32) u) of S."""
    M = g.shape[0]
    p, S = product(g.T, x)
    return p, max(ACC, (M + 32) * U32) * S + F32 * p.abs()


def colsum_bounds(g):
    """(ref, tol) of ga_linear_bias_grad_bf16: the fp32 sum of each column, at most 32 terms per warp, 8 warps per
    chunk and ceil(M / 256) chunks deep."""
    M = g.shape[0]
    depth = min(M, 32) + 8 + (M + 255) // 256
    gd = g.double()
    return gd.sum(0), depth * U32 * gd.abs().sum(0) + F32 * gd.sum(0).abs()


def check(got, ref, tol, what=""):
    """'' when every element of got is within its bound (NaN never is), else a message."""
    err = (got.double() - ref).abs()
    bad = ~(err <= tol)
    if not bool(bad.any()):
        return ""
    i = int(bad.flatten().nonzero()[0, 0])
    return "%s: %d elements outside their bound, first flat index %d: got %r want %r tol %r" % (
        what, int(bad.sum()), i, float(got.flatten()[i]), float(ref.flatten()[i]), float(tol.flatten()[i]))
