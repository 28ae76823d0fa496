"""fp64 references of the two tensor-core kernels (torch only; no library import), per-element error bounds, and
sentinel-filled buffers that show whether a kernel wrote outside its output.

GEMM  ga_gemm_bf16_tn: Y = A W^T + bias on the operands' exact bf16 values in float64, S = |A| |W|^T + |bias| (the
      magnitude of the summed terms), and each epilogue applied to Y in float64.
ATTN  ga_attention_bf16 / ga_attention_causal_bf16: O = softmax(scale Q K^T) V and P over the real keys only (keys
      above the query row masked too when causal), in float64, in query chunks.

Per-element bounds instead of one relative L2 norm: a single wrong element, a missing bias in one column or one
out-of-range key moves a large output's rel-L2 by far less than any useful threshold, but breaks its own element's
bound.  The constants come from the kernels' arithmetic, not from measurement:
  ACC = 2^-12      fp32 accumulation over K (and the fp32 bias add) relative to S.  The classic bound is K u S with
                   u = 2^-24; K <= 4096 on every call site.
  F32 = 2^-23      fp32 output rounding (and the gate product / residual add) relative to the result.
  BF16 = 2^-8      bf16 output rounding (round to nearest: half of one ulp of 2^-7) relative to the result.
  GELU' = 1.13     the largest |gelu'(x)| (1.1289 at x = 1.41): an error d in the GELU input moves the output by
                   at most 1.13 d.  GELU_APPROX = 2^-17 covers the kernel's erf (Abramowitz-Stegun 7.1.28,
                   |error| < 3e-7, plus the fp32 evaluation of (1 + ...)^-16 and one rcp.approx) as an absolute
                   error of at most 2^-17 |x| in gelu(x).
  q, k RMSNorm     first order: out_i = w_i y_i / rms, so |d out_i| <= |w_i| / rms (|d y_i| + |y_i / rms|
                   sum_j |y_j / rms| |d y_j| / 64); NORM_ARITH = 2^-16 relative for the fp32 sum of squares and rsqrt.
  attention        2^-7 (P |V|) for P rounded to bf16 in P V while l sums the unrounded fp32 probabilities (one bf16
                   rounding per term, times two for ex2.approx and the fp32 scores), + 2^-8 |O| for the bf16 output,
                   + 2^-16 max|V| as an absolute floor.

Set TC_REF_REPORT to a file path to have every check append one JSON line with its group and largest |err| / bound.
"""
import json
import math
import os

import torch

ACC = 2.0 ** -12
F32 = 2.0 ** -23
BF16 = 2.0 ** -8
GELU_D = 1.13
GELU_APPROX = 2.0 ** -17
NORM_ARITH = 2.0 ** -16
ATTN_P = 2.0 ** -7
ATTN_FLOOR = 2.0 ** -16

# GA_EPI_* of include/ga_b200.h
BF16_OUT, GELU_OUT, F32_OUT, RESID_GATE, HEADS, GEGLU = 0, 1, 2, 3, 4, 5

# Sentinels: signalling-NaN payloads.  GPU arithmetic and float -> bf16 conversion only ever produce the canonical
# NaN (0x7fffffff / 0x7fff), so a sentinel still in place was not written.
SENTINEL = {torch.float32: (torch.int32, 0x7FA5A5A5), torch.bfloat16: (torch.int16, 0x7FA5)}
# hostile padding values (the attention header requires finite padding)
K_PAD, VT_PAD, Q_PAD = 30.0, 1.0e4, 30.0


def _gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


# ---- guarded buffers ---------------------------------------------------------------------------------------------

class GuardBuf:
    """A tensor of `shape` inside a flat buffer with `slack` elements before and after it, every element set to the
    dtype's sentinel.  `t` is the tensor the kernel gets; intact(written) checks, bit for bit, that nothing outside
    the elements `written` marks (a bool tensor of `shape`, or None for nothing) changed, slack included."""

    def __init__(self, shape, dtype, device, slack=64):
        self.shape, self.dtype, self.slack = tuple(shape), dtype, slack
        self.n = math.prod(self.shape)
        self.ity, self.bits = SENTINEL[dtype]
        self.buf = torch.empty(self.n + 2 * slack, dtype=dtype, device=device)
        self.buf.view(self.ity).fill_(self.bits)
        self.t = self.buf[slack:slack + self.n].view(self.shape)

    def fill_outside(self, written):
        """Resets everything outside `written` to the sentinel (for a repeat call)."""
        bits = self.buf.view(self.ity)
        keep = bits.clone()
        bits.fill_(self.bits)
        if written is not None:
            inner = bits[self.slack:self.slack + self.n].view(self.shape)
            inner[written] = keep[self.slack:self.slack + self.n].view(self.shape)[written]

    def intact(self, written):
        """(ok, message): every element outside `written` still holds the sentinel."""
        bad = self.buf.view(self.ity) != self.bits
        if written is not None:
            bad[self.slack:self.slack + self.n].view(self.shape)[written] = False
        nbad = int(bad.sum())
        if nbad == 0:
            return True, ""
        first = int(bad.nonzero()[0, 0]) - self.slack
        where = "slack" if first < 0 or first >= self.n else "element %s" % (tuple(_unravel(first, self.shape)),)
        return False, "%d guard elements overwritten, first at %s" % (nbad, where)


def _unravel(i, shape):
    out = []
    for s in reversed(shape):
        out.append(i % s)
        i //= s
    return list(reversed(out))


def region(shape, *index, device=None):
    """A bool tensor of `shape`, True on t[index] (index: slices / ints as for tensor indexing)."""
    m = torch.zeros(shape, dtype=torch.bool, device=device)
    m[index] = True
    return m


def hostile_operand(rows, K, device, gen, scale=1.0, ld_extra=8, rows_extra=8):
    """A bf16 GEMM operand [rows, K] inside a [rows + rows_extra, K + ld_extra] buffer whose other elements are NaN:
    the kernel must never read them (the TMA box zero-fills the K tail and the rows past `rows`).
    Returns (buffer, view [rows, K], ld)."""
    ld = K + ld_extra
    buf = torch.full((rows + rows_extra, ld), float("nan"), dtype=torch.bfloat16, device=device)
    buf[:rows, :K] = (torch.randn(rows, K, generator=gen) * scale).to(device).to(torch.bfloat16)
    return buf, buf[:rows, :K], ld


# ---- GEMM ----------------------------------------------------------------------------------------------------------

def gemm_ref(A, W, bias=None):
    """A [M, K], W [N, K] (bf16 views), bias [N] fp32 or None -> (Y, S) float64 [M, N] on A's device."""
    a, w = A.double(), W.double()
    Y = a @ w.T
    S = a.abs() @ w.abs().T
    if bias is not None:
        Y += bias.double()
        S += bias.double().abs()
    return Y, S


def epilogue_ref(mode, Y, S, x0=None, gate=None):
    """(ref, tol) float64 of an element-wise epilogue on Y [M, N] (modes BF16_OUT, GELU_OUT, F32_OUT, RESID_GATE,
    GEGLU).  RESID_GATE: x0 [M, N] the residual before the call, gate [M, N] the gate each element sees (None = 1).
    GEGLU: columns (2j, 2j + 1) are (x_j, gate_j); the result has N / 2 columns."""
    if mode == BF16_OUT:
        ref = Y
        return ref, ACC * S + (BF16 + F32) * ref.abs()
    if mode == GELU_OUT:
        ref = _gelu(Y)
        return ref, GELU_D * ACC * S + GELU_APPROX * Y.abs() + (BF16 + F32) * ref.abs()
    if mode == F32_OUT:
        return Y, ACC * S + F32 * Y.abs()
    if mode == RESID_GATE:
        g = torch.ones_like(Y) if gate is None else gate.double()
        ref = x0.double() + g * Y
        return ref, ACC * S * g.abs() + F32 * ref.abs()
    if mode == GEGLU:
        x, gt, Sx, Sg = Y[:, 0::2], Y[:, 1::2], S[:, 0::2], S[:, 1::2]
        gg = _gelu(gt)
        ref = x * gg
        tol = ACC * (Sx * gg.abs() + GELU_D * x.abs() * Sg) + GELU_APPROX * x.abs() * gt.abs() + (BF16 + F32) * ref.abs()
        return ref, tol
    raise ValueError(mode)


def heads_ref(Y, S, B, rpb, heads, first_part, qn_w=None, kn_w=None, eps=1e-5):
    """HEADS epilogue of Y [B * rpb, N] ("(K H 64)" columns starting at part first_part).  Returns {part: (ref,
    tol)} with q, k as [B, heads, rpb, 64] and v as Vt [B, heads, 64, rpb], float64."""
    inner = heads * 64
    parts = Y.shape[1] // inner
    out = {}
    for p in range(parts):
        which = first_part + p
        y = Y[:, p * inner:(p + 1) * inner].reshape(B, rpb, heads, 64).permute(0, 2, 1, 3)
        s = S[:, p * inner:(p + 1) * inner].reshape(B, rpb, heads, 64).permute(0, 2, 1, 3)
        if which == 2:
            out["v"] = (y.transpose(-1, -2), (ACC * s + (BF16 + F32) * y.abs()).transpose(-1, -2))
            continue
        w = qn_w if which == 0 else kn_w
        if w is None:
            ref, tol = y, ACC * s + (BF16 + F32) * y.abs()
        else:
            w = w.double()
            rms = torch.sqrt(y.pow(2).mean(-1, keepdim=True) + eps)
            yh = y / rms
            ref = yh * w
            spread = (yh.abs() * s).sum(-1, keepdim=True) / 64.0
            tol = ACC * w.abs() / rms * (s + yh.abs() * spread) + (BF16 + NORM_ARITH) * ref.abs()
        out["q" if which == 0 else "k"] = (ref, tol)
    return out


# ---- attention -----------------------------------------------------------------------------------------------------

def attention_ref(q, k, vt, B, H, Nq, Nk, scale, causal=False, rows=None, chunk=512):
    """q [B*H, >= Nq, 64], k [B*H, >= Nk, 64], vt [B*H, 64, >= Nk] (the kernel's bf16 inputs).  rows: the query
    indices to compute (default all).  Returns (O, tol) float64 [B, len(rows), H * 64] (the kernel's output
    layout restricted to those rows)."""
    dev = q.device
    rows = torch.arange(Nq, device=dev) if rows is None else rows.to(dev)
    O = torch.empty(B * H, rows.numel(), 64, dtype=torch.float64, device=dev)
    T = torch.empty_like(O)
    for bh in range(B * H):
        kk = k[bh, :Nk].double()
        v = vt[bh, :, :Nk].double().T
        vmax = float(v.abs().max())
        for c0 in range(0, rows.numel(), chunk):
            r = rows[c0:c0 + chunk]
            s = (q[bh, r].double() @ kk.T) * scale
            if causal:
                s.masked_fill_(torch.arange(Nk, device=dev)[None, :] > r[:, None], float("-inf"))
            p = torch.softmax(s, dim=-1)
            o = p @ v
            O[bh, c0:c0 + chunk] = o
            T[bh, c0:c0 + chunk] = ATTN_P * (p @ v.abs()) + BF16 * o.abs() + ATTN_FLOOR * vmax
    fold = lambda t: t.view(B, H, -1, 64).permute(0, 2, 1, 3).reshape(B, -1, H * 64)
    return fold(O), fold(T)


def attention_inputs(B, H, Nq, Nk, pitch_q, pitch_k, device, gen, qk_scale=1.2):
    """Q, K, Vt of the kernel's layout with hostile padding: Q rows past Nq = Q_PAD, K rows past Nk = +-K_PAD with
    random signs (so that some padded key of a block scores high against every query), Vt columns past Nk = VT_PAD;
    all finite, as the header requires.  A padded key that is not masked, or a padded query row that leaks into a
    real one, moves the result by orders of magnitude."""
    q = torch.full((B * H, pitch_q, 64), Q_PAD, dtype=torch.bfloat16, device=device)
    sign = torch.randint(0, 2, (B * H, pitch_k, 64), generator=gen).to(device) * 2 - 1
    k = (sign * K_PAD).to(torch.bfloat16)
    vt = torch.full((B * H, 64, pitch_k), VT_PAD, dtype=torch.bfloat16, device=device)
    q[:, :Nq] = (torch.randn(B * H, Nq, 64, generator=gen) * qk_scale).to(device).to(torch.bfloat16)
    k[:, :Nk] = (torch.randn(B * H, Nk, 64, generator=gen) * qk_scale).to(device).to(torch.bfloat16)
    vt[:, :, :Nk] = torch.randn(B * H, 64, Nk, generator=gen).to(device, torch.bfloat16)
    return q, k, vt


def static_bound(q, k, Nq, Nk, scale):
    """A valid score bound: max |q| max |k| * scale over the real rows (Cauchy-Schwarz)."""
    return float(q[:, :Nq].double().norm(dim=-1).max() * k[:, :Nk].double().norm(dim=-1).max()) * scale


# ---- the check -----------------------------------------------------------------------------------------------------

def check(got, ref, tol, group="", what=""):
    """(max |err| / tol, message): message is empty when every element of got is within its bound (NaN never is)."""
    err = (got.double() - ref).abs()
    ratio = err / tol
    bad = ~(err <= tol)
    worst = float(torch.nan_to_num(ratio, nan=float("inf")).max()) if ratio.numel() else 0.0
    path = os.environ.get("TC_REF_REPORT")
    if path and group:
        with open(path, "a") as f:
            f.write(json.dumps({"group": group, "what": what, "max_ratio": worst}) + "\n")
    if not bool(bad.any()):
        return worst, ""
    idx = tuple(int(i) for i in bad.nonzero()[0])
    return worst, "%s: %d of %d elements outside the bound, first at %s: got %r want %r tol %.3g (max |err|/tol %.3g)" % (
        what, int(bad.sum()), bad.numel(), idx, float(got[idx]), float(ref[idx]), float(tol[idx]), worst)
