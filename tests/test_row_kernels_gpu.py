"""The networks' row-wise and element-wise kernels (include/ga_b200.h Parts 2, 3 and 5: norms, small linears, the DiT
prologue and final layer, token assembly, conversions) called one by one through the C ABI and compared element by
element with fp64 references written from the header's formulas, at the model shapes and on both sides of every
fast path: rows kept in registers (D % 4 == 0, D <= 1024) or not, the weight-prefetch path of ga_linear_small
(K % 128 == 0, K <= 1024) or not, row counts around a CTA's 8 rows and batch boundaries inside a CTA.

Every output buffer is followed by a guard tail (NaN, or an int16 sentinel for bf16) that must come back untouched.
Every entry point is called twice on the same inputs and must give the same bits: the kernels use no atomics.

Bounds are per element.  u = 2^-24; mag is the same expression evaluated on the absolute values of its operands, K
the length of the longest chain of fp32 roundings behind the element.  An fp32 result is held to |got - ref| <=
c u K mag, c = 2; a bf16 result may also differ by 2^-8 |ref|, its own rounding.  rsqrtf, expf, tanhf and
sinf / cosf add their documented ulp errors to K (__expf's 2 + 1.16 |x| ulp for SiLU).  A LayerNorm also carries the
error of its rounded fp32 mean, u K mean(|x|) rstd |w| per element: a row whose |mean| / std is about 100 is covered
without loosening the bound of the other rows.  Where a kernel rounds at most once per element its result is
replayed in fp32 or bf16 and must match bit for bit."""
import ctypes as C
import math
import zlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
U = 2.0 ** -24
BF = 2.0 ** -8
CF = 2.0                                    # the c of the bounds
PAD = 40                                    # guard-tail elements
GUARD16 = 0x7F7F
GELU_K0, GELU_K1 = 0.7978845608028654, 0.044715


# ---- plumbing ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def L():
    from gaussiananything_b200 import _lib
    return _lib.lib()


def _p(t):
    return C.c_void_p(t.data_ptr() if t is not None else 0)


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class Out:
    """A device buffer of n elements (`.t`) followed by a PAD-element guard tail."""

    def __init__(self, n, dtype=torch.float32, init=None):
        self.n, self.dtype = n, dtype
        if dtype == torch.bfloat16:
            self.full = torch.full((n + PAD,), GUARD16, dtype=torch.int16, device=DEV).view(torch.bfloat16)
        else:
            self.full = torch.full((n + PAD,), float("nan"), dtype=dtype, device=DEV)
        self.t = self.full[:n]
        if init is not None:
            self.t.copy_(init.reshape(-1))

    def tail_ok(self):
        tail = self.full[self.n:]
        if self.dtype == torch.bfloat16:
            return bool(torch.all(tail.view(torch.int16) == GUARD16))
        return bool(torch.all(torch.isnan(tail)))


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def twice(launch):
    """launch() allocates fresh guarded buffers, calls an entry point (which must return 0) and returns {name: Out}.
    It runs twice; every guard tail must be untouched and both runs must give the same bits.  Returns the first."""
    a = launch()
    torch.cuda.synchronize()
    b = launch()
    torch.cuda.synchronize()
    for k in a:
        assert a[k].tail_ok() and b[k].tail_ok(), "%s: guard tail overwritten" % k
        assert torch.equal(_bits(a[k].t), _bits(b[k].t)), "%s: two calls on the same inputs differ" % k
    return a


_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    """After the module: the largest |got - ref| / bound seen per entry point (shown with pytest -s)."""
    yield
    for k in sorted(_WORST):
        print("worst |got - ref| / bound  %-14s %.3g" % (k, _WORST[k]))


def within(got, ref, bound, what):
    """|got - ref| <= bound element by element (got finite); the message names the worst element."""
    got, ref, bound = got.double(), ref.double(), bound.double()
    assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
    assert bool(torch.isfinite(got).all()), "%s: non-finite output" % what
    r = (got - ref).abs() / bound.clamp_min(1e-300)
    i = int(torch.argmax(r))
    idx = np.unravel_index(i, tuple(r.shape))
    worst = float(r.reshape(-1)[i])
    _WORST[what.split(" ")[0]] = max(_WORST.get(what.split(" ")[0], 0.0), worst)
    assert worst <= 1.0, "%s: element %s got %.9g want %.9g bound %.3g" % (
        what, tuple(int(v) for v in idx), float(got.reshape(-1)[i]), float(ref.reshape(-1)[i]),
        float(bound.reshape(-1)[i]))


def same_bits(got, want, what):
    """Bit-for-bit equality; the message names the first differing element."""
    g, w = _bits(got), _bits(want.to(got.dtype))
    assert g.shape == w.shape, (what, tuple(g.shape), tuple(w.shape))
    bad = (g != w).nonzero()
    assert bad.numel() == 0, "%s: %d elements differ, first %s got %r want %r" % (
        what, bad.shape[0], tuple(bad[0].tolist()), got[tuple(bad[0])].item(), want[tuple(bad[0])].item())


def _gen(*key):
    return torch.Generator(device=DEV).manual_seed(zlib.crc32(repr(key).encode()))


def _randn(shape, g, scale=1.0, shift=0.0):
    return torch.randn(shape, device=DEV, generator=g) * scale + shift


def _silu(v):
    return v / (1 + torch.exp(-v))


def _silu_k(v):
    """K of fp32 x / (1 + __expf(-x)): __expf's 2 + 1.16 |x| ulp (2u each) and two roundings."""
    return 2 * (2 + 1.16 * v.abs()) + 2


def _gelu(v):
    return 0.5 * v * (1 + torch.tanh(GELU_K0 * (v + GELU_K1 * v ** 3)))


def _gelu_err(v, e_in):
    """Bound of |fp32 gelu_tanh(v + e) - gelu_tanh(v)| for an input error e_in: the slope (<= 1.13) times e_in, plus
    gelu_tanh's own roundings: the argument's five (relative to |k0 (v + k1 v^3)|, through tanh' <= 1), tanhf's 2 ulp,
    the final three."""
    a = (GELU_K0 * (v.abs() + GELU_K1 * v.abs() ** 3))
    return 1.13 * e_in + CF * U * (0.5 * v.abs() * (5 * a + 4) + 3 * _gelu(v).abs())


def _ln_ref(x, eps):
    """fp64 LayerNorm without affine: (n, rstd, mean(|x|) per row)."""
    xd = x.double()
    mu = xd.mean(-1, keepdim=True)
    var = ((xd - mu) ** 2).mean(-1, keepdim=True)
    rs = 1 / (var + eps).sqrt()
    return (xd - mu) * rs, rs, xd.abs().mean(-1, keepdim=True)


def _ln_k(D):
    """(K of the normalised element, K of the mean): the fp32 sums run D / 32 deep per lane, then 5 butterfly levels
    and a division; the variance adds a subtraction and a square per term; rsqrtf's 2 ulp, the division and eps."""
    Km = D / 32 + 8
    return Km / 2 + 12, Km


# ---- ga_rmsnorm_modulate --------------------------------------------------------------------------------------------
# (R, rows_per_batch, modulation): R % 8 of 5, 7 and 1; batches of 3 and 5 rows start inside CTAs
RMS_ROWS = [(5, 5, "none"), (263, 3, "chunks 0/1"), (257, 5, "chunks 3/4"), (15, 15, "none")]


@pytest.mark.parametrize("R,rpb,mode", RMS_ROWS, ids=["R%d rpb%d %s" % c for c in RMS_ROWS])
@pytest.mark.parametrize("D", [4, 768, 1024, 1028, 1152, 2048])
def test_rmsnorm_modulate(L, D, R, rpb, mode):
    """RMSNorm(x) w [(1 + scale[b]) + shift[b]] -> bf16, shift and scale chunks of a [B, 6 D] table at mod_ld 6 D as
    the DiT passes them.  |got - ref| <= 2 u K mag + 2^-8 |ref|, mag = |x rs w| (1 + |scale|) + |shift|, K = D / 64 +
    16 (half the D / 32 + 6 deep sum of squares through the square root, rsqrtf's 2 ulp, the division and eps, two
    products, the three modulation roundings)."""
    g = _gen("rms", D, R, rpb, mode)
    x = _randn((R, D), g, 2.0, 0.1)
    w = _randn((D,), g, 0.3, 1.0)
    B = -(-R // rpb)
    table = _randn((B, 6 * D), g, 0.5)
    eps = 1e-6
    if mode == "none":
        sh = sc = None
    else:
        c0 = 0 if mode == "chunks 0/1" else 3
        sh, sc = table[:, c0 * D:], table[:, (c0 + 1) * D:]

    def launch():
        o = Out(R * D, torch.bfloat16)
        assert L.ga_rmsnorm_modulate(_p(x), _p(w), _p(sh), _p(sc), 6 * D if sh is not None else 0, rpb, _p(o.t), R, D,
                                     eps, _st()) == 0
        return {"out": o}

    o = twice(launch)["out"]
    xd = x.double()
    rs = 1 / ((xd ** 2).mean(-1, keepdim=True) + eps).sqrt()
    y = xd * rs * w.double()
    mag = y.abs()
    if sh is not None:
        b = torch.arange(R, device=DEV) // rpb
        shd, scd = sh[:, :D].double()[b], sc[:, :D].double()[b]
        y = y * (1 + scd) + shd
        mag = mag * (1 + scd.abs()) + shd.abs()
    within(o.t.reshape(R, D), y, CF * U * (D / 64 + 16) * mag + BF * y.abs(), "rmsnorm D%d" % D)


# ---- ga_layernorm_modulate ------------------------------------------------------------------------------------------
LNM_MODES = ["affine", "w only", "per-token mod", "per-batch mod"]


@pytest.mark.parametrize("mode", LNM_MODES)
@pytest.mark.parametrize("D", [4, 64, 768, 1024])
def test_layernorm_modulate(L, D, mode):
    """LayerNorm(x) [w + b] [(1 + scale[b]) + shift[b]] -> bf16.  Affine (DINOv2, CLIP, the decoder's sr norms), w only,
    no affine with per-token shift / scale at mod_ld 6 depth D (the VAE decoder, depth 2), no affine with
    rows_per_batch 5.  Rows 1 and R - 1 have |mean| / std = 100.  |got - ref| <= 2 u (K mag + Km mean(|x|) rs |w|
    (1 + |scale|)) + 2^-8 |ref|, mag = (|n w| + |b|) (1 + |scale|) + |shift|, (K, Km) from _ln_k plus 5 roundings."""
    R = 263
    g = _gen("lnm", D, mode)
    x = _randn((R, D), g, 1.5, 0.2)
    x[1] = _randn((D,), g, 1.0, 100.0)
    x[R - 1] = _randn((D,), g, 1.0, -100.0)
    eps = 1e-6
    w = _randn((D,), g, 0.3, 1.0) if mode in ("affine", "w only") else None
    b = _randn((D,), g, 0.3) if mode == "affine" else None
    rpb, mod_ld, sh, sc = 1, 0, None, None
    if mode.endswith("mod"):
        depth = 2
        rpb = 1 if mode == "per-token mod" else 5
        nb = R if rpb == 1 else -(-R // rpb)
        mod_ld = 6 * depth * D
        table = _randn((nb, mod_ld), g, 0.5)
        sh, sc = table[:, 6 * D:], table[:, 7 * D:]            # layer 1's chunks 0 and 1

    def launch():
        o = Out(R * D, torch.bfloat16)
        assert L.ga_layernorm_modulate(_p(x), _p(w), _p(b), _p(sh), _p(sc), mod_ld, rpb, _p(o.t), R, D, eps,
                                       _st()) == 0
        return {"out": o}

    o = twice(launch)["out"]
    n, rs, am = _ln_ref(x, eps)
    wd = w.double() if w is not None else torch.ones(D, dtype=torch.float64, device=DEV)
    bd = b.double() if b is not None else torch.zeros(D, dtype=torch.float64, device=DEV)
    y = n * wd + bd
    mag = (n * wd).abs() + bd.abs()
    mterm = am * rs * wd.abs()
    if sh is not None:
        bi = torch.arange(R, device=DEV) // rpb
        shd, scd = sh[:, :D].double()[bi], sc[:, :D].double()[bi]
        y = y * (1 + scd) + shd
        mag = mag * (1 + scd.abs()) + shd.abs()
        mterm = mterm * (1 + scd.abs())
    K, Km = _ln_k(D)
    within(o.t.reshape(R, D), y, CF * U * ((K + 5) * mag + Km * mterm) + BF * y.abs(), "ln_modulate D%d %s" % (D, mode))


# ---- ga_layernorm_rows ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("affine", ["none", "w", "w+b"])
@pytest.mark.parametrize("D", [4, 768, 1024, 1, 3, 770, 1025, 1152])
def test_layernorm_rows(L, D, affine):
    """fp32 LayerNorm [* w [+ b]], 17 rows; D in {4, 768, 1024} keeps the row in registers, the others take the
    three-pass loop.  Rows 1 and 16 have |mean| / std = 100.  |got - ref| <= 2 u (K mag + Km mean(|x|) rs |w|), mag =
    |n w| + |b|, (K, Km) from _ln_k plus 2 roundings."""
    R = 17
    g = _gen("lnr", D, affine)
    x = _randn((R, D), g, 1.5, -0.3)
    x[1] = _randn((D,), g, 1.0, 100.0)
    x[16] = _randn((D,), g, 1.0, -100.0)
    w = _randn((D,), g, 0.3, 1.0) if affine != "none" else None
    b = _randn((D,), g, 0.3) if affine == "w+b" else None
    eps = 1e-5

    def launch():
        o = Out(R * D)
        assert L.ga_layernorm_rows(_p(x), _p(w), _p(b), _p(o.t), R, D, eps, _st()) == 0
        return {"y": o}

    o = twice(launch)["y"]
    n, rs, am = _ln_ref(x, eps)
    wd = w.double() if w is not None else torch.ones(D, dtype=torch.float64, device=DEV)
    bd = b.double() if b is not None else torch.zeros(D, dtype=torch.float64, device=DEV)
    y = n * wd + bd
    K, Km = _ln_k(D)
    within(o.t.reshape(R, D), y, CF * U * ((K + 2) * ((n * wd).abs() + bd.abs()) + Km * am * rs * wd.abs()),
           "ln_rows D%d %s" % (D, affine))


# ---- ga_linear_small ------------------------------------------------------------------------------------------------
LS_K = [128, 256, 768, 1024, 1, 129, 300, 1152]
LS_ACT = [(a, b, c) for a in (0, 1) for b in (0, 1) for c in (0, 1)]


@pytest.mark.parametrize("act_in,act_out,acc", LS_ACT, ids=["in%d out%d acc%d" % a for a in LS_ACT])
@pytest.mark.parametrize("K", LS_K)
def test_linear_small(L, K, act_in, act_out, acc):
    """y (+)= act_out(bias + act_in(x) W^T): SiLU on the sum, then the old y added.  Rows 1, 2, 15 or 16 and N 57 or 63
    (N % 8 of 1 and 7) in turn; bias NULL in every other case.  |got - ref| <= e, e_lin = 2 u K (|act_in(x)| |W|^T +
    |bias|), K = K / 32 + 8 (+ the input SiLU's K, at most 6 + 2.32 max|x|); with act_out e = 1.1 e_lin + 2 u
    K_silu(s) |silu(s)|; accumulate adds 2 u |ref|."""
    i = LS_K.index(K) + LS_ACT.index((act_in, act_out, acc))
    rows, N = (1, 2, 15, 16)[i % 4], (57, 63)[i % 2]
    g = _gen("ls", K, act_in, act_out, acc)
    x = _randn((rows, K), g)
    W = _randn((N, K), g, 1 / math.sqrt(K))
    bias = _randn((N,), g, 0.5) if i % 2 == 0 else None
    y0 = _randn((rows, N), g)

    def launch():
        o = Out(rows * N, init=y0 if acc else None)
        assert L.ga_linear_small(_p(x), _p(W), _p(bias), _p(o.t), rows, N, K, act_in, act_out, acc, _st()) == 0
        return {"y": o}

    o = twice(launch)["y"]
    xd = x.double()
    xa = _silu(xd) if act_in else xd
    bd = bias.double() if bias is not None else torch.zeros(N, dtype=torch.float64, device=DEV)
    s = xa @ W.double().t() + bd
    Kd = K / 32 + 8 + (float(_silu_k(xd).max()) if act_in else 0)
    e = CF * U * Kd * (xa.abs() @ W.double().abs().t() + bd.abs())
    ref = s
    if act_out:
        ref = _silu(s)
        e = 1.1 * e + CF * U * _silu_k(s) * ref.abs()
    if acc:
        ref = ref + y0.double()
        e = e + CF * U * ref.abs()
    within(o.t.reshape(rows, N), ref, e, "linear_small K%d rows%d N%d" % (K, rows, N))


# ---- ga_final_layer -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Cout", [1, 3, 10, 16])
@pytest.mark.parametrize("D", [4, 768, 1024, 770, 1152])
def test_final_layer(L, D, Cout):
    """bias + (LayerNorm(x) (1 + scale[b]) + shift[b]) W^T, eps 1e-6, 37 rows in batches of 5 (boundaries inside the
    CTAs' 8 rows); Cout 10 is the point DiTs' latent width.  h = n (1 + scale) + shift carries e_h = 2 u ((K + 3)
    |h|m + Km mean(|x|) rs (1 + |scale|)), |h|m = |n| (1 + |scale|) + |shift|; |got - ref| <= e_h |W|^T + 2 u (D / 32 +
    7) (|h|m |W|^T + |bias|)."""
    R, rpb = 37, 5
    B = -(-R // rpb)
    g = _gen("final", D, Cout)
    x = _randn((R, D), g, 1.5, 0.4)
    x[9] = _randn((D,), g, 1.0, 100.0)
    mod = _randn((B, 2, D), g, 0.4)
    W = _randn((Cout, D), g, 1 / math.sqrt(D))
    bias = _randn((Cout,), g, 0.3)
    eps = 1e-6

    def launch():
        o = Out(R * Cout)
        assert L.ga_final_layer(_p(x), _p(mod), _p(W), _p(bias), _p(o.t), R, D, Cout, rpb, eps, _st()) == 0
        return {"y": o}

    o = twice(launch)["y"]
    n, rs, am = _ln_ref(x, eps)
    bi = torch.arange(R, device=DEV) // rpb
    sh, sc = mod[:, 0].double()[bi], mod[:, 1].double()[bi]
    h = n * (1 + sc) + sh
    hm = n.abs() * (1 + sc.abs()) + sh.abs()
    K, Km = _ln_k(D)
    e_h = CF * U * ((K + 3) * hm + Km * am * rs * (1 + sc.abs()))
    Wd = W.double()
    ref = h @ Wd.t() + bias.double()
    bound = e_h @ Wd.abs().t() + CF * U * (D / 32 + 7) * (hm @ Wd.abs().t() + bias.double().abs())
    within(o.t.reshape(R, Cout), ref, bound, "final_layer D%d Cout%d" % (D, Cout))


# ---- ga_timestep_sinusoid -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", [2, 256, 2048])
def test_timestep_sinusoid(L, dim):
    """[cos(t f_i) | sin(t f_i)], f_i = exp(-ln(1e4) i / half), t in {0, 1e-4, 0.5, 1, 999, 1000, -3}.  The fp32
    argument a_i = -ln(1e4) i / half carries three roundings (logf's 1 ulp, the product, the division), so
    |a_i - exact| <= 3 u |a_i|; expf turns that absolute error into a relative one and adds its 2 ulp: f_i's relative
    error is <= (3 |a_i| + 4) u (|a_i| <= ln 1e4).  t f_i adds one rounding, and cosf / sinf their 2 ulp.  So |got -
    ref| <= 2 u ((3 |a_i| + 5) |t f_i| + 2 |ref|); t = 0 gives cos 1 and sin 0 exactly."""
    half = dim // 2
    t = torch.tensor([0.0, 1e-4, 0.5, 1.0, 999.0, 1000.0, -3.0], device=DEV)
    rows = t.numel()

    def launch():
        o = Out(rows * dim)
        assert L.ga_timestep_sinusoid(_p(t), _p(o.t), rows, dim, _st()) == 0
        return {"out": o}

    o = twice(launch)["out"].t.reshape(rows, dim)
    i = torch.arange(half, device=DEV, dtype=torch.float64)
    a = -math.log(1e4) * i / half
    arg = t.double()[:, None] * torch.exp(a)[None]
    ref = torch.cat([torch.cos(arg), torch.sin(arg)], 1)
    k = (3 * a.abs() + 5)[None] * arg.abs()
    bound = CF * U * (torch.cat([k, k], 1) + 2 * ref.abs())
    within(o, ref, bound, "sinusoid dim%d" % dim)
    assert torch.equal(o[0, :half], torch.ones_like(o[0, :half])) and torch.equal(_bits(o[0, half:]),
                                                                                   _bits(torch.zeros_like(o[0, half:])))


# ---- ga_add_tables --------------------------------------------------------------------------------------------------
# (what, L, rows, JD, t0_ld)
ADD = [("dit D1024", 24, 2, 6 * 1024, 6 * 1024), ("dit D768 B3", 3, 3, 6 * 768, 6 * 768),
       ("final-layer broadcast D1024", 1, 3, 2 * 1024, 1024), ("final-layer broadcast D4", 1, 5, 8, 4)]


@pytest.mark.parametrize("what,Ln,rows,JD,t0_ld", ADD, ids=[a[0] for a in ADD])
def test_add_tables(L, what, Ln, rows, JD, t0_ld):
    """mod[l, b, e] = tables[l, e] + t0[b, e % t0_ld], one fp32 addition: bit for bit against torch's fp32 addition.
    The final layer's call (JD = 2 t0_ld) gives both halves the same temb.  t0 is followed by one more row, so a wrong
    index reads numbers rather than past the allocation."""
    g = _gen("add", what)
    tables = _randn((Ln, JD), g)
    t0_full = _randn((rows + 1, t0_ld), g)

    def launch():
        o = Out(Ln * rows * JD)
        assert L.ga_add_tables(_p(tables), _p(t0_full), _p(o.t), Ln, rows, JD, t0_ld, _st()) == 0
        return {"mod": o}

    o = twice(launch)["mod"].t.reshape(Ln, rows, JD)
    t0 = t0_full[:rows].repeat(1, JD // t0_ld)
    same_bits(o, tables[:, None, :] + t0[None], what)


# ---- ga_embed_fc1 ---------------------------------------------------------------------------------------------------
# (what, Cx, C2, D, R): the point DiTs (stage 1: 3 channels; stage 2: 10 latent channels after the 3 fps xyz), the
# decoder's post_quant fc1 (zc 10, pq_k a multiple of 16), Cx = 1; R D % 256 != 0 where D allows it
EMB = [("stage1 D1024", 3, 0, 1024, 37), ("stage2 concat D1024", 10, 3, 1024, 37), ("stage2 concat D768", 10, 3, 768, 5),
       ("post_quant pq_k 208", 10, 0, 208, 35), ("Cx1 concat D100", 1, 3, 100, 3), ("Cx1 D768", 1, 0, 768, 1)]


@pytest.mark.parametrize("what,Cx,C2,D,R", EMB, ids=[e[0] for e in EMB])
def test_embed_fc1(L, what, Cx, C2, D, R):
    """bf16(gelu_tanh(b1 + W1 [xin2 | xin])) against fp64 tanh-GELU of the fp64 sum: |got - ref| <= _gelu_err(v,
    2 u (Cx + C2 + 1) mag) + 2^-8 |ref|, mag = |b1| + |W1| [|xin2| | |xin|]."""
    g = _gen("emb", what)
    xin = _randn((R, Cx), g)
    xin2 = _randn((R, C2), g) if C2 else None
    W1 = _randn((D, C2 + Cx), g, 0.7)
    b1 = _randn((D,), g, 0.3)

    def launch():
        o = Out(R * D, torch.bfloat16)
        assert L.ga_embed_fc1(_p(xin), Cx, _p(xin2), C2, _p(W1), _p(b1), _p(o.t), R, D, _st()) == 0
        return {"h": o}

    o = twice(launch)["h"]
    inp = torch.cat([xin2, xin], 1) if C2 else xin
    v = inp.double() @ W1.double().t() + b1.double()
    mag = inp.double().abs() @ W1.double().abs().t() + b1.double().abs()
    ref = _gelu(v)
    within(o.t.reshape(R, D), ref, _gelu_err(v, CF * U * (Cx + C2 + 1) * mag) + BF * ref.abs(), "embed_fc1 " + what)


# ---- ga_xyz_posenc --------------------------------------------------------------------------------------------------
def _bf16_rn64(v):
    """int16 bits of the bf16 round-to-nearest-even of fp64 v, rounded once: fp32 round-to-odd first (exact for the
    second rounding, 24 bits > 8 + 2), then to bf16."""
    f = v.float()
    b = f.view(torch.int32)
    b = torch.where(f.double().abs() > v.abs(), b - 1, b)                 # toward zero: the truncated fp32
    b = torch.where(b.view(torch.float32).double() != v, b | 1, b)        # inexact: set the sticky bit
    u = b.long() & 0xFFFFFFFF
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) & 0xFFFF
    return torch.where(r >= 0x8000, r - 0x10000, r).to(torch.int16)


def _bf16_key(bits16):
    """int16 bf16 bits -> an integer that orders the values (+0 and -0 both 0)."""
    u = bits16.int() & 0xFFFF
    return torch.where(u < 0x8000, u, -(u - 0x8000))


@pytest.mark.parametrize("R", [1, 127, 128, 129, 4097])
def test_xyz_posenc(L, R):
    """[x, sin(2^k x), cos(2^k x)]_{k < 10}, 63 features and a zero column.  The first rows hold 0, +-1 and +-4, so
    the arguments reach 4 * 2^9 = 2048.  2^k x is exact in fp32 and sinf / cosf are within 2 ulp, so each feature is
    the bf16 rounding of the fp64 value or its neighbour; columns 0-2 are bf16(x) exactly and column 63 is +0."""
    g = _gen("pe", R)
    xyz = _randn((R, 3), g, 1.5)
    special = torch.tensor([[0.0, 1.0, -1.0], [4.0, -4.0, 0.0], [-4.0, 0.0, 4.0]], device=DEV)
    n = min(R, 3)
    xyz[:n] = special[:n]

    def launch():
        o = Out(R * 64, torch.bfloat16)
        assert L.ga_xyz_posenc(_p(xyz), _p(o.t), R, _st()) == 0
        return {"pe": o}

    o = twice(launch)["pe"].t.reshape(R, 64)
    xd = xyz.double()
    cols = [xd]
    for k in range(10):
        cols += [torch.sin(xd * 2.0 ** k), torch.cos(xd * 2.0 ** k)]
    ref = torch.cat(cols, 1)                                               # [R, 63]
    same_bits(o[:, :3], xyz.to(torch.bfloat16), "posenc xyz columns")
    d = (_bf16_key(_bits(o[:, 3:63])) - _bf16_key(_bf16_rn64(ref[:, 3:]))).abs()
    bad = (d > 1).nonzero()
    assert bad.numel() == 0, "posenc: element %s got %r want %r" % (
        tuple(bad[0].tolist()), o[:, 3:63][tuple(bad[0])].item(), ref[:, 3:][tuple(bad[0])].item())
    assert bool((_bits(o[:, 63]) == 0).all()), "posenc: column 63 is not +0"


# ---- ga_cfg_combine, ga_axpy ----------------------------------------------------------------------------------------
SIZES = [1, 255, 257, 3_000_001]


def _fma_or_not(got, base, s, d, what):
    """got = base + s d for fp32 base, s, d: either the unfused fp32 replay fp32(base + fp32(s d)), bit for bit, or the
    fused one, base + s d rounded once (within half an ulp of the exact value).  Under cancellation the two differ by
    many ulps of the result, so neither a one-ulp bound around the unfused value nor one around the fused value would
    hold for both."""
    g = got.cpu().numpy()
    b, dd = base.cpu().numpy(), d.cpu().numpy()
    s32 = np.float32(s)
    unfused = b + s32 * dd                                                  # numpy fp32: each operation rounded
    p = np.float64(s32) * dd.astype(np.float64)                             # exact: 24 + 24 bits
    S = p + b.astype(np.float64)
    bb = S - p
    err = (p - (S - bb)) + (b.astype(np.float64) - bb)                      # S + err = p + base exactly
    fused_ok = np.abs((g.astype(np.float64) - S) - err) <= 0.5 * np.spacing(np.abs(g)).astype(np.float64)
    ok = (g.view(np.int32) == unfused.view(np.int32)) | fused_ok
    bad = np.flatnonzero(~ok)
    assert bad.size == 0, "%s: element %d got %.9g, unfused %.9g, exact %.12g" % (
        what, bad[0], g[bad[0]], unfused[bad[0]], S[bad[0]] + err[bad[0]])


@pytest.mark.parametrize("s", [0.0, 1.0, 4.5])
@pytest.mark.parametrize("n", SIZES)
def test_cfg_combine(L, n, s):
    """h = u + s (c - u) written to both halves, same bits in both; with d = fp32(c - u), h is u + s d either unfused or
    contracted into one FMA (_fma_or_not); s = 0 returns u exactly."""
    g = _gen("cfg", n, s)
    eps = _randn((2 * n,), g)

    def launch():
        o = Out(2 * n)
        assert L.ga_cfg_combine(_p(eps), _p(o.t), n, s, _st()) == 0
        return {"out": o}

    o = twice(launch)["out"].t
    assert torch.equal(_bits(o[:n]), _bits(o[n:])), "cfg: the two halves differ"
    c, u = eps[:n], eps[n:]
    if s == 0.0:
        same_bits(o[:n], u, "cfg s=0")
    else:
        _fma_or_not(o[:n], u, s, c - u, "cfg s=%g" % s)


@pytest.mark.parametrize("a", [0.0, 0.37, -2.0])
@pytest.mark.parametrize("n", SIZES)
def test_axpy(L, n, a):
    """x += a v, either unfused or contracted into one FMA (_fma_or_not); a = 0 leaves x's bits unchanged."""
    g = _gen("axpy", n, a)
    x0, v = _randn((n,), g), _randn((n,), g, 3.0)

    def launch():
        o = Out(n, init=x0)
        assert L.ga_axpy(_p(o.t), _p(v), a, n, _st()) == 0
        return {"x": o}

    o = twice(launch)["x"].t
    if a == 0.0:
        same_bits(o, x0, "axpy a=0")
    else:
        _fma_or_not(o, x0, a, v, "axpy a=%g" % a)


# ---- ga_f32_to_bf16, ga_silu_to_bf16 --------------------------------------------------------------------------------
def test_f32_to_bf16(L):
    """Bit for bit against torch's round-to-nearest-even over ±0, subnormals, ties with even and odd bf16 mantissas,
    values that round up into the next binade, FLT_MAX (to inf), ±inf, and a million random bit patterns; NaN stays
    NaN."""
    special = [0x00000000, 0x80000000, 0x00000001, 0x80000001, 0x007FFFFF, 0x00008000, 0x00018000, 0x00800000,
               0x3F808000, 0x3F818000, 0xBF808000, 0xBF818000, 0x3F808001, 0x3F817FFF, 0x3F7FFFFF, 0x3F7F8000,
               0x3F7F7FFF, 0xBF7FFFFF, 0x7F7FFFFF, 0xFF7FFFFF, 0x7F7F8000, 0x7F7F7FFF, 0x7F800000, 0xFF800000,
               0x7FC00000, 0xFFC00000, 0x7F800001, 0x7FFFFFFF]
    g = torch.Generator().manual_seed(zlib.crc32(b"f2b"))
    rnd = torch.randint(-2 ** 31, 2 ** 31 - 1, (1 << 20,), generator=g, dtype=torch.int64)
    bits = torch.cat([torch.tensor(special, dtype=torch.int64), rnd])
    bits = torch.where(bits >= 2 ** 31, bits - 2 ** 32, bits).to(torch.int32)
    x = bits.view(torch.float32).to(DEV)
    n = x.numel()

    def launch():
        o = Out(n, torch.bfloat16)
        assert L.ga_f32_to_bf16(_p(x), _p(o.t), n, _st()) == 0
        return {"y": o}

    o = twice(launch)["y"].t
    nan = torch.isnan(x)
    assert bool(torch.isnan(o[nan]).all()), "f32_to_bf16: a NaN did not stay NaN"
    same_bits(o[~nan], x[~nan].cpu().to(torch.bfloat16).to(DEV), "f32_to_bf16")


def test_silu_to_bf16(L):
    """bf16(x / (1 + __expf(-x))) against fp64 SiLU: |got - ref| <= 2 u K_silu(x) |ref| + 2^-8 |ref| + 2^-120.  Inputs
    span +-12 and include large negatives (-20 ... -1e4): below x = -88.7 the fp32 exp(-x) overflows and the kernel
    returns -0 where the exact value is below 2^-120 in magnitude, which the absolute term allows."""
    g = _gen("silu")
    x = torch.cat([_randn((1 << 16,), g, 4.0), torch.linspace(-12, 12, 4097, device=DEV),
                   torch.tensor([-20.0, -50.0, -80.0, -87.0, -88.0, -88.7, -89.0, -100.0, -1e4, 30.0, 1e4, 0.0],
                                device=DEV)])
    n = x.numel()

    def launch():
        o = Out(n, torch.bfloat16)
        assert L.ga_silu_to_bf16(_p(x), _p(o.t), n, _st()) == 0
        return {"y": o}

    o = twice(launch)["y"].t
    xd = x.double()
    ref = _silu(xd)
    within(o, ref, CF * U * _silu_k(xd) * ref.abs() + BF * ref.abs() + 2.0 ** -120, "silu_to_bf16")


# ---- ga_thin_linear -------------------------------------------------------------------------------------------------
THIN = [(R, Cc, ln, silu) for R in (17, 31) for Cc in (1, 13, 16) for ln in (0, 1) for silu in (0, 1)]


@pytest.mark.parametrize("R,Cc,ln,silu", THIN, ids=["R%d C%d ln%d silu%d" % t for t in THIN])
def test_thin_linear(L, R, Cc, ln, silu):
    """y = bias + f(x) W^T, f = [LayerNorm affine] then [SiLU]; R odd (R % 16 of 1 and 15: the last warp has one row
    of its two), D 768, 1024 or 64 in turn, bias NULL in every other case.  The guard tail after y must stay NaN.
    h = f(x) carries e_h (the LayerNorm bound of test_layernorm_rows, then 1.1 e + 2 u K_silu |silu| through the
    SiLU); |got - ref| <= e_h |W|^T + 2 u (D / 32 + 7) (|h| |W|^T + |bias|)."""
    i = THIN.index((R, Cc, ln, silu))
    D = (768, 1024, 64)[i % 3]
    g = _gen("thin", R, Cc, ln, silu)
    x = _randn((R, D), g, 1.5, 0.3)
    x[R - 1] = _randn((D,), g, 1.0, 50.0)
    lw, lb = (_randn((D,), g, 0.3, 1.0), _randn((D,), g, 0.3)) if ln else (None, None)
    W = _randn((Cc, D), g, 1 / math.sqrt(D))
    bias = _randn((Cc,), g, 0.3) if i % 2 == 0 else None
    eps = 1e-6

    def launch():
        o = Out(R * Cc)
        assert L.ga_thin_linear(_p(x), _p(lw), _p(lb), silu, _p(W), _p(bias), _p(o.t), R, D, Cc, eps, _st()) == 0
        return {"y": o}

    o = twice(launch)["y"]
    if ln:
        n, rs, am = _ln_ref(x, eps)
        K, Km = _ln_k(D)
        h = n * lw.double() + lb.double()
        e_h = CF * U * ((K + 2) * ((n * lw.double()).abs() + lb.double().abs()) + Km * am * rs * lw.double().abs())
    else:
        h = x.double()
        e_h = torch.zeros_like(h)
    if silu:
        s = _silu(h)
        e_h = 1.1 * e_h + CF * U * _silu_k(h) * s.abs()
        h = s
    bd = bias.double() if bias is not None else torch.zeros(Cc, dtype=torch.float64, device=DEV)
    Wd = W.double()
    ref = h @ Wd.t() + bd
    bound = e_h @ Wd.abs().t() + CF * U * (D / 32 + 7) * (h.abs() @ Wd.abs().t() + bd.abs())
    within(o.t.reshape(R, Cc), ref, bound, "thin_linear R%d C%d D%d" % (R, Cc, D))


# ---- ga_micro_seq_build ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [768, 4])
def test_micro_seq_build(L, D):
    """The deployed cascade's sequences chained stage after stage: f = 8 from the 5 parent tokens (prev_f 0), then
    f = 4 from stage 1's sequence buffer (prev_f 8), then f = 3 from stage 2's (prev_f 4).  Pure copies, bit for bit
    against torch indexing of the previous stage's buffer."""
    g = _gen("seq", D)
    parents = _randn((5, D), g)
    S, prev_f, prev_seq = 5, 0, parents
    for f in (8, 4, 3):
        q = _randn((f, D), g)

        def launch():
            o = Out(S * (1 + f) * D)
            assert L.ga_micro_seq_build(_p(prev_seq), prev_f, _p(q), _p(o.t), S, f, D, _st()) == 0
            return {"seq": o}

        seq = twice(launch)["seq"].t.reshape(S, 1 + f, D)
        s = torch.arange(S, device=DEV)
        if prev_f == 0:
            head = prev_seq[s]
        else:
            head = prev_seq.reshape(S // prev_f, 1 + prev_f, D)[s // prev_f, 1 + s % prev_f]
        want = torch.cat([head[:, None], q[None].expand(S, f, D)], 1)
        same_bits(seq, want, "seq build f%d prev_f%d" % (f, prev_f))
        prev_seq, prev_f, S = seq.reshape(-1, D).clone(), f, S * f


# ---- ga_dino_tokens -------------------------------------------------------------------------------------------------
DINO = [(4, 1369, 1024, 2), (0, 1369, 1024, 1), (4, 4, 4, 3), (0, 4, 4, 2), (4, 4, 1024, 3), (0, 1369, 4, 3)]


@pytest.mark.parametrize("n_reg,n_patch,D,batch", DINO, ids=["reg%d patch%d D%d B%d" % d for d in DINO])
def test_dino_tokens(L, n_reg, n_patch, D, batch):
    """cls + pos[0] | registers (no pos_embed) | patch_out + pos[1 + j]: one fp32 addition or a copy per element, bit
    for bit against torch."""
    g = _gen("dino", n_reg, n_patch, D, batch)
    pe = _randn((batch * n_patch, D), g)
    cls = _randn((D,), g)
    reg = _randn((n_reg, D), g) if n_reg else None
    pos = _randn((1 + n_patch, D), g)
    nt = 1 + n_reg + n_patch

    def launch():
        o = Out(batch * nt * D)
        assert L.ga_dino_tokens(_p(pe), _p(cls), _p(reg), n_reg, _p(pos), _p(o.t), batch, n_patch, D, _st()) == 0
        return {"x": o}

    o = twice(launch)["x"].t.reshape(batch, nt, D)
    parts = [(cls + pos[0]).expand(batch, 1, D)]
    if n_reg:
        parts.append(reg[None].expand(batch, n_reg, D))
    parts.append(pe.reshape(batch, n_patch, D) + pos[1:][None])
    same_bits(o, torch.cat(parts, 1), "dino tokens")


# ---- ga_vae_enc_input -----------------------------------------------------------------------------------------------
# (what, n, C, c_pad, H, W, step, off, token_xyz)
ENC_IN = [("encoder 27x41 8/4", 2, 15, 16, 27, 41, 8, 4, True), ("encoder 33x20 1/0", 2, 15, 16, 33, 20, 1, 0, True),
          ("encoder 27x41 off 26", 1, 15, 16, 27, 41, 8, 26, True), ("disc 27x41", 3, 3, 8, 27, 41, 0, 0, False),
          ("disc 20x33 xyz 1/0", 2, 3, 8, 20, 33, 1, 0, True), ("disc 33x20 off 19", 2, 3, 8, 33, 20, 3, 19, True)]


@pytest.mark.parametrize("what,n,Cc,c_pad,H,W,step,off,txyz", ENC_IN, ids=[e[0] for e in ENC_IN])
def test_vae_enc_input(L, what, n, Cc, c_pad, H, W, step, off, txyz):
    """x_bf16 NHWC = bf16(img), the padding channels exactly +0; token_xyz = img[:, C-3:C, off::step, off::step] in
    (n ty tx) order, copied bit for bit.  A call with bad token arguments (off = min(H, W)) returns GA_ERR_BADARG and
    writes neither output.  img is followed by one more image, so a wrong index reads numbers rather than past the
    allocation."""
    g = _gen("encin", what)
    img = _randn((n + 1, Cc, H, W), g, 2.0)[:n]
    xyz_c = Cc - 3
    Ht = (H - off + step - 1) // step if txyz else 0
    Wt = (W - off + step - 1) // step if txyz else 0

    def launch():
        o = {"x": Out(n * H * W * c_pad, torch.bfloat16)}
        if txyz:
            o["t"] = Out(n * Ht * Wt * 3)
        assert L.ga_vae_enc_input(_p(img), n, Cc, H, W, c_pad, _p(o["x"].t), xyz_c, step, off,
                                  _p(o["t"].t) if txyz else None, _st()) == 0
        return o

    o = twice(launch)
    want = torch.zeros(n, H, W, c_pad, dtype=torch.bfloat16, device=DEV)
    want[..., :Cc] = img.permute(0, 2, 3, 1).to(torch.bfloat16)
    same_bits(o["x"].t.reshape(n, H, W, c_pad), want, what + " x_bf16")
    if txyz:
        tw = img[:, xyz_c:xyz_c + 3, off::step, off::step].permute(0, 2, 3, 1).reshape(-1, 3)
        same_bits(o["t"].t.reshape(-1, 3), tw, what + " token_xyz")
        bx, bt = Out(n * H * W * c_pad, torch.bfloat16), Out(n * Ht * Wt * 3)
        assert L.ga_vae_enc_input(_p(img), n, Cc, H, W, c_pad, _p(bx.t), xyz_c, step, min(H, W), _p(bt.t),
                                  _st()) == -1
        torch.cuda.synchronize()
        assert bool((bx.full.view(torch.int16) == GUARD16).all()), "x_bf16 written by a refused call"
        assert bool(torch.isnan(bt.full).all()), "token_xyz written by a refused call"


# ---- ga_vae_enc_head ------------------------------------------------------------------------------------------------
def _head_weights(D, hid, zc, g, big):
    """fp32 weights of the readout head; `big` gives quant_conv fc2's logvar rows biases of +-150 and small weights, so
    |moments| >= 100."""
    w = dict(ln_w=_randn((D,), g, 0.2, 1.0), ln_b=_randn((D,), g, 0.2),
             fc1_w=_randn((hid, D), g, 1 / math.sqrt(D)), fc1_b=_randn((hid,), g, 0.2),
             fc2_w=_randn((2 * zc, hid), g, 1 / math.sqrt(hid)), fc2_b=_randn((2 * zc,), g, 0.2),
             q1_w=_randn((2 * zc, 2 * zc), g, 1 / math.sqrt(2 * zc)), q1_b=_randn((2 * zc,), g, 0.2),
             q2_w=_randn((2 * zc, 2 * zc), g, 1 / math.sqrt(2 * zc)), q2_b=_randn((2 * zc,), g, 0.2))
    if big:
        w["q2_w"][zc:] *= 0.1
        w["q2_b"][zc:] = torch.where(w["q2_b"][zc:] >= 0, 150.0, -150.0)
    return w


def _head_struct(w, eps):
    from gaussiananything_b200._lib import GaVaeEncHead
    names = ("ln_w", "ln_b", "fc1_w", "fc1_b", "fc2_w", "fc2_b", "q1_w", "q1_b", "q2_w", "q2_b")
    return GaVaeEncHead(*[w[k].data_ptr() for k in names], eps)


def _head_check(o, x, noise, w, D, hid, zc, eps, what):
    """h_out against fp64 from x: the LayerNorm bound, then through each layer e_out = e_in |W|^T + 2 u (n_in + 1)
    (|in| |W|^T + |b|) (one fmaf chain per output) and _gelu_err.  mean, logvar, std and latent against fp64 from the
    kernel's own h_out: the same for quant_conv; logvar = 20 tanh(m / 20) adds (1 - tanh^2) e_m and 2 u (3 |logvar| +
    |m / 20| ...) for the division and tanhf's 2 ulp; std = exp(logvar / 2) adds std (e_lv / 2 + 2 u 4); latent = mean
    + std noise adds e_mean + |noise| e_std + 2 u (|latent| + |std noise|)."""
    what = "head " + what
    Wd = {k: v.double() for k, v in w.items()}
    n, rs, am = _ln_ref(x, eps)
    K, Km = _ln_k(D)
    xn = n * Wd["ln_w"] + Wd["ln_b"]
    e = CF * U * ((K + 2) * ((n * Wd["ln_w"]).abs() + Wd["ln_b"].abs()) + Km * am * rs * Wd["ln_w"].abs())

    def layer(v, e, Wn, bn, n_in, act):
        s = v @ Wd[Wn].t() + Wd[bn]
        es = e @ Wd[Wn].abs().t() + CF * U * (n_in + 1) * (v.abs() @ Wd[Wn].abs().t() + Wd[bn].abs())
        return (_gelu(s), _gelu_err(s, es)) if act else (s, es)

    hv, e = layer(xn, e, "fc1_w", "fc1_b", D, True)
    h, e = layer(hv, e, "fc2_w", "fc2_b", hid, False)
    within(o["h"].t.reshape(-1, 2 * zc), h, e, what + " h_out")
    hk = o["h"].t.reshape(-1, 2 * zc).double()
    q1, e = layer(hk, torch.zeros_like(hk), "q1_w", "q1_b", 2 * zc, True)
    q2, e = layer(q1, e, "q2_w", "q2_b", 2 * zc, False)
    m, lvin, e_m, e_in = q2[:, :zc], q2[:, zc:], e[:, :zc], e[:, zc:]
    within(o["mean"].t.reshape(-1, zc), m, e_m, what + " mean")
    th = torch.tanh(lvin / 20)
    lv = 20 * th
    e_lv = (1 - th ** 2) * e_in + CF * U * (3 * lv.abs() + (1 - th ** 2) * lvin.abs())
    within(o["logvar"].t.reshape(-1, zc), lv, e_lv, what + " logvar")
    sd = torch.exp(lv / 2)
    e_sd = sd * (e_lv / 2 + CF * U * 4)
    if "std" in o:
        within(o["std"].t.reshape(-1, zc), sd, e_sd, what + " std")
    if "latent" in o:
        nz = noise.double() if noise is not None else torch.zeros_like(m)
        lat = m + sd * nz
        within(o["latent"].t.reshape(-1, zc), lat, e_m + nz.abs() * e_sd + CF * U * (lat.abs() + (sd * nz).abs()),
               what + " latent")
    return lvin


# (what, R, D, hid, zc, noise, std and latent, saturated moments)
HEAD = [("encoder 256 zc10", 9, 256, 512, 10, True, True, False),
        ("encoder 256 zc10 saturated", 9, 256, 512, 10, True, True, True),
        ("D200 hid300 no noise", 5, 200, 300, 10, False, True, True),
        ("D300 hid200 std latent NULL", 5, 300, 200, 10, True, False, False),
        ("D513 hid129", 3, 513, 129, 7, True, True, True)]


@pytest.mark.parametrize("what,R,D,hid,zc,with_noise,outs,big", HEAD, ids=[h[0] for h in HEAD])
def test_vae_enc_head(L, what, R, D, hid, zc, with_noise, outs, big):
    """The readout head split at h_out (bounds in _head_check).  D and hid below and above 256 and not multiples of it,
    so the CTA's strided loops end in a partial pass; noise NULL (latent = mean); stdv and latent NULL; quant_conv
    weights that drive |moments| >= 100 so the soft clamp 20 tanh(m / 20) saturates."""
    g = _gen("head", what)
    eps = 1e-6
    w = _head_weights(D, hid, zc, g, big)
    x = _randn((R, D), g, 1.5, 0.3)
    noise = _randn((R, zc), g) if with_noise else None
    p = _head_struct(w, eps)

    def launch():
        o = dict(h=Out(R * 2 * zc), mean=Out(R * zc), logvar=Out(R * zc))
        if outs:
            o.update(std=Out(R * zc), latent=Out(R * zc))
        assert L.ga_vae_enc_head(C.byref(p), _p(x), _p(noise), R, D, hid, zc, _p(o["h"].t), _p(o["mean"].t),
                                 _p(o["logvar"].t), _p(o["std"].t) if outs else None,
                                 _p(o["latent"].t) if outs else None, _st()) == 0
        return o

    o = twice(launch)
    lvin = _head_check(o, x, noise, w, D, hid, zc, eps, what)
    if big:
        assert float(lvin.abs().min()) >= 100, "the moments do not reach the soft clamp's saturation"


def test_vae_enc_head_smem_limit(L):
    """(D + hid + 6 zc) 4 bytes of dynamic shared memory plus the kernel's 32 static bytes: the largest size the host
    accepts, 49 152 bytes in all, launches and computes the head (bounds in _head_check); one float more is
    GA_ERR_SIZE."""
    zc, hid = 2, 268
    D = (48 * 1024 - 32) // 4 - hid - 6 * zc
    g = _gen("head limit")
    w = _head_weights(D, hid, zc, g, False)
    x = _randn((2, D), g, 1.5, 0.3)
    p = _head_struct(w, 1e-6)

    def launch(D_call=D):
        o = dict(h=Out(2 * 2 * zc), mean=Out(2 * zc), logvar=Out(2 * zc))
        rc = L.ga_vae_enc_head(C.byref(p), _p(x), None, 2, D_call, hid, zc, _p(o["h"].t), _p(o["mean"].t),
                               _p(o["logvar"].t), None, None, _st())
        return rc, o

    rc, _ = launch(D + 1)
    assert rc == -3, "one float past the limit: got %d, want GA_ERR_SIZE" % rc

    def ok():
        rc, o = launch()
        assert rc == 0, "the largest accepted size does not launch: %d" % rc
        return o

    o = twice(ok)
    _head_check(o, x, None, w, D, hid, zc, 1e-6, "head at the limit")


