"""PatchGAN discriminator kernels (include/ga_b200.h Part 11) called one by one through the C ABI and compared element
by element with fp64 references of the same operation on the same bf16 / fp32 operands, at the model's layer shapes
for 24 x 24, 27 x 41, 50 x 70, 64 x 64 and 4 x 512^2 images and at the edges of the 128-row tiles.

Every output and partial buffer is followed by a guard tail (NaN, or an int16 sentinel for bf16) that must come back
untouched; partial buffers are sized exactly by the row counts the library reports and must be written in full.
Every entry point is called twice on the same inputs and must give the same bits: the kernels use no atomics.

Bounds are per element.  u = 2^-24; mag is the same operation on the absolute values of the operands (the sum of the
|terms|), K the length of the longest fp32 chain of roundings behind the element.  An fp32 result is held to
|got - ref| <= c u K mag, c = 2 (the tensor cores may truncate where fp32 rounds); a bf16 result adds 2^-8 |ref|, its
own rounding.  Where the header fixes every fp32 operation (BatchNorm's apply kernels), the result is replayed in
fp32 numpy from the kernel's own statistics and must match bit for bit."""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gaussiananything_b200 import disc
from oracle import disc_oracle as do

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
U = 2.0 ** -24
BF = 2.0 ** -8
CF = 2.0                                    # the c of the bounds
SLOPE = float(np.float32(0.2))              # the kernels' 0.2f
PAD = 40                                    # guard-tail elements
GUARD16 = 0x7F7F
SMALL = 50_000_000                          # multiply-adds under which the numpy oracle gives the reference


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


def within(got, ref, bound, what):
    """|got - ref| <= bound element by element (got finite); the message names the worst element."""
    got, ref, bound = got.double(), ref.double(), bound.double()
    assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
    assert bool(torch.isfinite(got).all()), "%s: non-finite output" % what
    r = (got - ref).abs() / bound.clamp_min(1e-300)
    i = int(torch.argmax(r))
    idx = np.unravel_index(i, tuple(r.shape))
    assert float(r.reshape(-1)[i]) <= 1.0, "%s: element %s got %.9g want %.9g bound %.3g" % (
        what, tuple(int(v) for v in idx), float(got.reshape(-1)[i]), float(ref.reshape(-1)[i]),
        float(bound.reshape(-1)[i]))


def _gen(*key):
    return torch.Generator(device=DEV).manual_seed(zlib.crc32(repr(key).encode()))


def _act(shape, g):
    """A LeakyReLU output in bf16: both signs, so every mask and epilogue branch is taken."""
    v = torch.randn(shape, device=DEV, generator=g)
    return torch.where(v > 0, v, SLOPE * v).to(torch.bfloat16)


def _nchw(t):
    """NHWC (bf16 or fp32) -> NCHW fp64."""
    return t.double().permute(0, 3, 1, 2)


def _rows(t):
    """NCHW -> [n H W, C]."""
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])


def _lrelu(v, mask=None):
    keep = (v if mask is None else mask) > 0
    return torch.where(keep, v, SLOPE * v)


def _np(fn, *ts, **kw):
    return torch.from_numpy(fn(*[t.cpu().numpy() for t in ts], **kw)).to(DEV)


def ref_conv(x, w, s):
    """4x4 pad-1 convolution, fp64; the numpy oracle for the small shapes."""
    Ho, Wo = do.out_size(x.shape[2], s), do.out_size(x.shape[3], s)
    if x.shape[0] * Ho * Wo * w.numel() < SMALL:
        return _np(do.conv, x, w, s=s)
    return F.conv2d(x, w, stride=s, padding=1)


def ref_dgrad(g, w, s, H, W):
    """d(sum g * conv(x)) / dx for x [n, Ci, H, W], fp64: the oracle's parity decomposition (stride 2) or scatter
    (stride 1) for the small shapes, torch's conv_transpose2d for the large ones."""
    if g.numel() * w.shape[1] * 16 < SMALL:
        if s == 2:
            return _np(do.conv_dgrad_parity, g, w, H=H, W=W)
        return _np(do.conv_dgrad, g, w, s=s, H=H, W=W)
    op = (H - (g.shape[2] - 1) * s - 2, W - (g.shape[3] - 1) * s - 2)
    return F.conv_transpose2d(g, w, stride=s, padding=1, output_padding=op)


def ref_wgrad(g, x, s):
    """d(sum g * conv(x)) / dW [Co, Ci, 4, 4], fp64."""
    if g.numel() * x.shape[1] * 16 < SMALL:
        return _np(do.conv_wgrad, g, x, s=s)
    Ho, Wo = g.shape[2], g.shape[3]
    xp = F.pad(x, (1, 1, 1, 1))
    dw = torch.empty(g.shape[1], x.shape[1], 4, 4, dtype=torch.float64, device=DEV)
    for ky in range(4):
        for kx in range(4):
            xs = xp[:, :, ky:ky + s * (Ho - 1) + 1:s, kx:kx + s * (Wo - 1) + 1:s]
            dw[:, :, ky, kx] = torch.einsum("nohw,nchw->oc", g, xs)
    return dw


def _bf16_bits(y32):
    """bf16 bits (round to nearest even) of an fp32 numpy array, as int16."""
    u = np.ascontiguousarray(y32, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return (((u + 0x7FFF + ((u >> 16) & 1)) >> 16) & 0xFFFF).astype(np.uint16).view(np.int16)


def _f32(t):
    return t.float().cpu().numpy()


# ---- ga_conv4x4_lrelu_bf16 ------------------------------------------------------------------------------------------
# (what, n, H, W, Cin, channels used, Cout): conv 1 at every image size (64 channels: the 64-wide tile), and a
# 128-channel output (the 128-wide tile)
LRELU = [("conv1 24x24", 2, 24, 24, 8, 3, 64), ("conv1 27x41", 2, 27, 41, 8, 3, 64),
         ("conv1 50x70", 4, 50, 70, 8, 3, 64), ("conv1 64x64", 4, 64, 64, 8, 3, 64),
         ("conv1 4x512", 4, 512, 512, 8, 3, 64), ("128 out 27x41", 2, 13, 20, 64, 64, 128),
         ("128 out 64x64", 2, 32, 32, 64, 64, 128)]


@pytest.mark.parametrize("what,n,H,W,cin,used,cout", LRELU, ids=[c[0] for c in LRELU])
def test_conv4x4_lrelu_bf16(L, what, n, H, W, cin, used, cout):
    """Stride 2, bias.  bf16(lrelu(bias + conv)) against fp64 conv + bias + LeakyReLU of the same bf16 operands (conv 1:
    channels 3-7 of the input and of the pack zero): |got - ref| <= 2 u K mag + 2^-8 |ref|, K = 16 Cin + 2 (the taps,
    the bias, the slope), mag = conv(|x|, |w|) + |bias|."""
    g = _gen("lrelu", what)
    x = torch.zeros(n, H, W, cin, device=DEV, dtype=torch.bfloat16)
    x[..., :used] = torch.randn(n, H, W, used, device=DEV, generator=g).to(torch.bfloat16)
    w = torch.randn(cout, used, 4, 4, device=DEV, generator=g) * 0.05
    b = torch.randn(cout, device=DEV, generator=g) * 0.2
    wp, kp = disc.pack_forward(w, cin)
    Ho, Wo = do.out_size(H, 2), do.out_size(W, 2)
    M = n * Ho * Wo

    def launch():
        o = Out(M * cout, torch.bfloat16)
        assert L.ga_conv4x4_lrelu_bf16(_p(x), n, H, W, cin, _p(wp), kp, _p(b), cout, 2, _p(o.t), _st()) == 0
        return {"out": o}

    o = twice(launch)["out"]
    x64, w64 = _nchw(x[..., :used]), w.to(torch.bfloat16).double()
    ref = _rows(_lrelu(ref_conv(x64, w64, 2) + b.double().reshape(1, -1, 1, 1)))
    mag = _rows(ref_conv(x64.abs(), w64.abs(), 2) + b.double().abs().reshape(1, -1, 1, 1))
    within(o.t.reshape(M, cout), ref, CF * U * (16 * cin + 2) * mag + BF * ref.abs(), what)


# ---- ga_conv4x4_stats ------------------------------------------------------------------------------------------------
# (what, n, H, W, Cin, Cout, stride): convs 2-4 at the layer shapes; M = n Ho Wo at the 128-row tile edges
STATS = [
    ("conv2 24x24", 4, 12, 12, 64, 128, 2),        # M 144
    ("conv2 27x41", 4, 13, 20, 64, 128, 2),        # M 240
    ("conv2 4x512", 4, 256, 256, 64, 128, 2),      # M 65536: 512 partials, four per finalize thread
    ("conv3 24x24 n57", 57, 6, 6, 128, 256, 2),    # M 513 = 4 * 128 + 1
    ("conv3 24x24 n71", 71, 6, 6, 128, 256, 2),    # M 639 = 4 * 128 + 127
    ("conv3 50x70", 4, 12, 17, 128, 256, 2),       # M 192
    ("conv3 64x64", 4, 16, 16, 128, 256, 2),       # M 256
    ("conv4 24x24", 4, 3, 3, 256, 512, 1),         # M 16
    ("conv4 27x41", 4, 3, 5, 256, 512, 1),         # M 32
    ("conv4 50x70 n11", 11, 6, 8, 256, 512, 1),    # M 385 = 3 * 128 + 1
    ("conv4 64x64", 4, 8, 8, 256, 512, 1),         # M 196
    ("conv4 M=2", 1, 2, 3, 256, 512, 1),           # M 2, BatchNorm's minimum
]
_STATS = {}


def _stats_run(L, case):
    """The stats kernel on case's inputs (twice, guard tails checked), cached for the BatchNorm tests."""
    what, n, H, W, cin, cout, s = case
    if what in _STATS:
        return _STATS[what]
    g = _gen("stats", what)
    x = _act((n, H, W, cin), g)
    w = torch.randn(cout, cin, 4, 4, device=DEV, generator=g) * 0.02
    wp, kp = disc.pack_forward(w, cin)
    Ho, Wo = do.out_size(H, s), do.out_size(W, s)
    M = n * Ho * Wo
    nb = -(-M // 128)

    def launch():
        z, part = Out(M * cout), Out(nb * cout * 2)
        assert L.ga_conv4x4_stats(_p(x), n, H, W, cin, _p(wp), kp, cout, s, _p(z.t), _p(part.t), _st()) == 0
        return {"z": z, "partial": part}

    r = twice(launch)
    _STATS[what] = dict(x=x, w=w, wp=wp, kp=kp, M=M, nb=nb, Ho=Ho, Wo=Wo, z=r["z"].t.reshape(M, cout),
                        partial=r["partial"].t.reshape(nb, cout, 2))
    return _STATS[what]


@pytest.mark.parametrize("case", STATS, ids=[c[0] for c in STATS])
def test_conv4x4_stats(L, case):
    """z against the fp64 convolution: |z - ref| <= 2 u K mag, K = 16 Cin.  Partial row b, over the cnt rows
    [128 b, 128 b + 128) of [0, M) of the kernel's own z: m_b against their fp64 mean, |m_b - mean| <= 2 u (cnt + 1)
    mean(|z|) (an fp32 sum and a division); M2_b against the fp64 sum of (z - m_b)^2 (the header's definition),
    |M2_b - ref| <= 2 u (cnt + 3) ref.  Every partial row is written, none past ceil(M / 128).  Without partials (eval
    mode) z has the same bits."""
    what, n, H, W, cin, cout, s = case
    r = _stats_run(L, case)
    M, nb, z, part = r["M"], r["nb"], r["z"], r["partial"]
    x64, w64 = _nchw(r["x"]), r["w"].to(torch.bfloat16).double()
    ref = _rows(ref_conv(x64, w64, s))
    mag = _rows(ref_conv(x64.abs(), w64.abs(), s))
    within(z, ref, CF * U * 16 * cin * mag, what + " z")
    # per partial row, against the kernel's own z
    zd = torch.zeros(nb * 128, cout, dtype=torch.float64, device=DEV)
    zd[:M] = z.double()
    valid = (torch.arange(nb * 128, device=DEV) < M).double().reshape(nb, 128, 1)
    cnt = valid.sum(1)                                           # [nb, 1]
    zb = zd.reshape(nb, 128, cout)
    mean = zb.sum(1) / cnt
    within(part[..., 0], mean, CF * U * (cnt + 1) * zb.abs().sum(1) / cnt, what + " partial mean")
    mb = part[..., 0].double().reshape(nb, 1, cout)
    m2 = (((zb - mb) * valid) ** 2).sum(1)
    within(part[..., 1], m2, CF * U * (cnt + 3) * m2, what + " partial M2")
    # eval mode: no partials, the same z
    z2 = Out(M * cout)
    assert L.ga_conv4x4_stats(_p(r["x"]), n, H, W, cin, _p(r["wp"]), r["kp"], cout, s, _p(z2.t), None, _st()) == 0
    torch.cuda.synchronize()
    assert z2.tail_ok() and torch.equal(_bits(z2.t), _bits(z.reshape(-1)))


# ---- ga_disc_bn_forward ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["train momentum 0.1", "train momentum 0.3", "eval"])
@pytest.mark.parametrize("case", STATS, ids=[c[0] for c in STATS])
def test_bn_forward(L, case, mode):
    """On the stats kernel's z and partials.  Training: mean against the fp64 mean of z, |got - ref| <= 2 u K mean(|z|),
    K = 130 (a 128-row fp32 sum, its division and the final rounding); rstd against fp64 1 / sqrt(var + eps) (biased
    var), |got - ref| <= 2 u K ref (1 + mean(|z|) / std), K = 260 (the fp32 M2 terms, and the per-CTA means' errors
    through Chan's cross terms); running mean fp32((1 - m) rm + m mean) and running var fp32((1 - m) rv + m var M /
    (M - 1)) within m times those bounds plus 2 u |ref|.  Eval: mean_out is the running mean and rstd_out
    fp32(1 / sqrt(rv + eps)) in fp64, bit for bit, and the running statistics keep their bits.  Both: a_out bit for bit
    against bf16(lrelu(((z - mean) rstd) gamma + beta)) replayed in fp32 numpy from the kernel's mean_out and
    rstd_out."""
    what, n, H, W, cin, cout, s = case
    r = _stats_run(L, case)
    M, z, part = r["M"], r["z"], r["partial"]
    training = mode != "eval"
    mom = float(np.float32(0.3 if "0.3" in mode else 0.1)) if training else 0.0
    eps = float(np.float32(1e-5))
    g = _gen("bnf", what, mode)
    gamma = 1 + 0.2 * torch.randn(cout, device=DEV, generator=g)
    beta = 0.2 * torch.randn(cout, device=DEV, generator=g)
    rm0 = 0.1 * torch.randn(cout, device=DEV, generator=g)
    rv0 = 0.5 + torch.rand(cout, device=DEV, generator=g)

    def launch():
        o = dict(rm=Out(cout, init=rm0), rv=Out(cout, init=rv0), mean=Out(cout), rstd=Out(cout),
                 a=Out(M * cout, torch.bfloat16))
        assert L.ga_disc_bn_forward(_p(z), _p(part) if training else None, M, cout, _p(gamma), _p(beta),
                                    int(training), mom, eps, _p(o["rm"].t), _p(o["rv"].t), _p(o["mean"].t),
                                    _p(o["rstd"].t), _p(o["a"].t), _st()) == 0
        return o

    o = twice(launch)
    mean_out, rstd_out = o["mean"].t, o["rstd"].t
    if training:
        zd = z.double()
        mu = zd.mean(0)
        var = zd.var(0, correction=0)
        absmean = zd.abs().mean(0)
        b_mean = CF * U * 130 * absmean
        rel_var = CF * U * 260 * (1 + absmean / var.sqrt())
        within(mean_out, mu, b_mean, what + " mean")
        rstd = 1 / (var + eps).sqrt()
        within(rstd_out, rstd, rel_var * rstd, what + " rstd")
        rm = (1 - mom) * rm0.double() + mom * mu
        rv = (1 - mom) * rv0.double() + mom * var * M / (M - 1)
        within(o["rm"].t, rm, mom * b_mean + 2 * U * rm.abs(), what + " running mean")
        within(o["rv"].t, rv, mom * 2 * rel_var * var * M / (M - 1) + 2 * U * rv.abs(), what + " running var")
    else:
        assert torch.equal(_bits(mean_out), _bits(rm0))
        want = (1.0 / np.sqrt(rv0.cpu().numpy().astype(np.float64) + eps)).astype(np.float32)
        assert np.array_equal(rstd_out.cpu().numpy().view(np.int32), want.view(np.int32))
        assert torch.equal(_bits(o["rm"].t), _bits(rm0)) and torch.equal(_bits(o["rv"].t), _bits(rv0))
    zz, mn, rs, ga, be = _f32(z), _f32(mean_out), _f32(rstd_out), _f32(gamma), _f32(beta)
    y = ((zz - mn) * rs) * ga + be
    y = np.where(y > 0, y, np.float32(SLOPE) * y)
    got = o["a"].t.view(torch.int16).cpu().numpy().reshape(M, cout)
    bad = np.argwhere(got != _bf16_bits(y))
    assert bad.size == 0, "%s a_out: %d elements differ from the fp32 replay, first %s" % (what, len(bad), bad[0])


# ---- ga_disc_conv5 --------------------------------------------------------------------------------------------------
# (what, n, H, W): conv 5's input at each image size; 2 x 2 has one output pixel, 2 x 4 one output row, 4 x 2 one
# output column
CONV5 = [("24x24", 2, 2, 2), ("27x41", 3, 2, 4), ("41x27", 3, 4, 2), ("50x70", 4, 5, 7), ("64x64", 4, 7, 7),
         ("4x512", 4, 63, 63)]


@pytest.mark.parametrize("what,n,H,W", CONV5, ids=[c[0] for c in CONV5])
def test_conv5(L, what, n, H, W):
    """Logits against the fp64 convolution of the bf16 input with the fp32 weights plus the bias: |got - ref| <=
    2 u K mag, K = 16 * 16 + 5 + 2 (a lane's 16 taps x 16 channels in sequence, the 5-level butterfly, the bias, the
    rounding of each product), mag = conv(|x|, |w|) + |bias|."""
    g = _gen("conv5", what)
    x = _act((n, H, W, 512), g)
    w5 = torch.randn(16, 512, device=DEV, generator=g) * 0.02
    b5 = torch.randn(1, device=DEV, generator=g) * 0.1
    Ho, Wo = H - 1, W - 1

    def launch():
        o = Out(n * Ho * Wo)
        assert L.ga_disc_conv5(_p(x), n, H, W, _p(w5), _p(b5), _p(o.t), _st()) == 0
        return {"logits": o}

    o = twice(launch)["logits"]
    W5 = w5.double().reshape(4, 4, 512).permute(2, 0, 1).unsqueeze(0)
    x64 = _nchw(x)
    ref = (ref_conv(x64, W5, 1) + b5.double()).reshape(-1)
    mag = (ref_conv(x64.abs(), W5.abs(), 1) + b5.double().abs()).reshape(-1)
    within(o.t, ref, CF * U * (16 * 16 + 5 + 2) * mag, what)


# ---- ga_disc_conv5_backward -----------------------------------------------------------------------------------------
# (what, n, H, W): P = n H W is never a multiple of 256
C5B = [("24x24", 2, 2, 2), ("27x41", 4, 2, 4), ("50x70", 4, 5, 7), ("64x64", 4, 7, 7), ("64x64 n9", 9, 7, 7),
       ("4x512", 4, 63, 63)]


@pytest.mark.parametrize("what,n,H,W", C5B, ids=[c[0] for c in C5B])
def test_conv5_backward(L, what, n, H, W):
    """gy4 against fp64 lrelu'(a4) * conv_transpose(g5, w5): |got - ref| <= 2 u K mag, K = 2 * 16 + 1 (16 rounded
    products and sums, the slope).  BN 4's partials summed over their ga_disc_conv5_partials rows (fp64) against the
    fp64 sums over pixels of gy and gy xhat (xhat = (z4 - mean4) rstd4): 2 u K sum(mag) and 2 u K sum(mag |xhat|),
    K = 33 + 256 + 3 (a 256-pixel fp32 sum, xhat's two roundings).  dw5 against the fp64 weight gradient:
    2 u K mag, K = 2 * 256 + 1 (rounded products summed in fp32 over a block's 256 pixels; the blocks in fp64).  gy4 and
    the partials have the same bits with and without dw5."""
    g = _gen("c5b", what)
    Ho, Wo = H - 1, W - 1
    P = n * H * W
    nb = L.ga_disc_conv5_partials(n, H, W)
    assert nb == -(-P // 256) and P % 256
    g5 = torch.randn(n, Ho, Wo, device=DEV, generator=g)
    w5 = torch.randn(16, 512, device=DEV, generator=g) * 0.02
    a4 = _act((n, H, W, 512), g)
    z4 = torch.randn(P, 512, device=DEV, generator=g) * 2 + 0.5
    mean4 = 0.5 + 0.1 * torch.randn(512, device=DEV, generator=g)
    rstd4 = 0.5 + 0.1 * torch.rand(512, device=DEV, generator=g)

    def launch(with_dw):
        o = dict(gy4=Out(P * 512), bn_partial=Out(nb * 512 * 2))
        if with_dw:
            o.update(dw_partial=Out(nb * 16 * 512), dw5=Out(16 * 512))
        dwp, dw5 = (o["dw_partial"].t, o["dw5"].t) if with_dw else (None, None)
        assert L.ga_disc_conv5_backward(_p(g5), n, H, W, _p(w5), _p(a4), _p(z4), _p(mean4), _p(rstd4),
                                        _p(o["gy4"].t), _p(o["bn_partial"].t), _p(dwp), _p(dw5), _st()) == 0
        return o

    o = twice(lambda: launch(True))
    o2 = twice(lambda: launch(False))
    for k in ("gy4", "bn_partial"):
        assert torch.equal(_bits(o[k].t), _bits(o2[k].t)), k + " depends on whether dw5 is formed"
    W5 = w5.double().reshape(4, 4, 512).permute(2, 0, 1).unsqueeze(0)
    g64 = g5.double().unsqueeze(1)
    mask = _rows(_nchw(a4))
    ga = _rows(ref_dgrad(g64, W5, 1, H, W))
    mag = _rows(ref_dgrad(g64.abs(), W5.abs(), 1, H, W))
    gy = _lrelu(ga, mask)
    within(o["gy4"].t.reshape(P, 512), gy, CF * U * 33 * mag, what + " gy4")
    part = o["bn_partial"].t.reshape(nb, 512, 2).double()
    assert bool(torch.isfinite(part).all()), "a partial row is not written"
    xhat = (z4.double() - mean4.double()) * rstd4.double()
    K = 33 + 256 + 3
    within(part[..., 0].sum(0), gy.sum(0), CF * U * K * mag.sum(0), what + " sum gy")
    within(part[..., 1].sum(0), (gy * xhat).sum(0), CF * U * K * (mag * xhat.abs()).sum(0), what + " sum gy xhat")
    a64 = _nchw(a4)
    dw = ref_wgrad(g64, a64, 1)[0].permute(1, 2, 0).reshape(16, 512)
    dwm = ref_wgrad(g64.abs(), a64.abs(), 1)[0].permute(1, 2, 0).reshape(16, 512)
    within(o["dw5"].t.reshape(16, 512), dw, CF * U * (2 * 256 + 1) * dwm, what + " dw5")


# ---- ga_disc_dgrad --------------------------------------------------------------------------------------------------
# (what, n, H, W, Cg, Cout, stride, bn): H x W is the dgrad's output, the forward convolution's input.  Conv 2's dgrad
# ends in conv 1's LeakyReLU (bf16 out), conv 3's and conv 4's in BatchNorm 2 and 3 (fp32 gy and partials).
DGRAD = [
    ("conv2 24x24", 2, 12, 12, 128, 64, 2, False),
    ("conv2 27x41", 2, 13, 20, 128, 64, 2, False),
    ("conv2 50x70", 2, 25, 35, 128, 64, 2, False),
    ("conv2 64x64", 2, 32, 32, 128, 64, 2, False),
    ("conv2 1x512", 1, 256, 256, 128, 64, 2, False),
    ("conv2 3x2", 2, 3, 2, 128, 64, 2, False),
    ("conv3 24x24", 4, 6, 6, 256, 128, 2, True),
    ("conv3 27x41", 4, 6, 10, 256, 128, 2, True),
    ("conv3 50x70", 4, 12, 17, 256, 128, 2, True),
    ("conv3 64x64", 4, 16, 16, 256, 128, 2, True),
    ("conv3 3x2", 2, 3, 2, 256, 128, 2, True),     # parity classes one row wide
    ("conv3 2x3", 2, 2, 3, 256, 128, 2, True),     # ... and one column wide
    ("conv3 2x2", 3, 2, 2, 256, 128, 2, True),
    ("bn 64-wide 7x9", 2, 7, 9, 128, 64, 2, True),
    ("conv4 24x24", 4, 3, 3, 512, 256, 1, True),
    ("conv4 24x24 n57", 57, 3, 3, 512, 256, 1, True),   # M 513
    ("conv4 27x41", 4, 3, 5, 512, 256, 1, True),
    ("conv4 50x70", 4, 6, 8, 512, 256, 1, True),
    ("conv4 64x64", 4, 8, 8, 512, 256, 1, True),
    ("lrelu stride 1 5x7", 2, 5, 7, 128, 64, 1, False),
]


def _dgrad_rows(n, H, W, s):
    """The partial rows the dgrad writes: one per 128-row CTA, for stride 2 of each parity class in turn."""
    if s == 1:
        return -(-n * H * W // 128)
    return sum(-(-n * ((H - py + 1) // 2) * ((W - px + 1) // 2) // 128) for py in range(2) for px in range(2))


@pytest.mark.parametrize("case", DGRAD, ids=[c[0] for c in DGRAD])
def test_dgrad(L, case):
    """Output against fp64 conv_transpose of the bf16 gradient with the bf16 weights, the LeakyReLU mask applied:
    |got - ref| <= 2 u K mag (+ 2^-8 |ref| for the bf16 output), K = 4 Cg + 1 (stride 2, a 2 x 2 parity kernel) or
    16 Cg + 1 (stride 1).  With BatchNorm, the partial rows, exactly ga_disc_dgrad_partials of them and all written,
    summed (fp64) against the fp64 sums over pixels of gy and gy xhat: 2 u K' sum(mag) and 2 u K' sum(mag |xhat|),
    K' = K + 128 + 3."""
    what, n, H, W, cg, cout, s, bn = case
    g = _gen("dgrad", what)
    Hg, Wg = do.out_size(H, s), do.out_size(W, s)
    M = n * H * W
    dz = torch.randn(n, Hg, Wg, cg, device=DEV, generator=g).to(torch.bfloat16)
    w = torch.randn(cg, cout, 4, 4, device=DEV, generator=g) * 0.03
    wf, kpf = disc.pack_dgrad(w, s)
    act = _act((n, H, W, cout), g)
    rows = L.ga_disc_dgrad_partials(n, H, W, s)
    assert rows == _dgrad_rows(n, H, W, s)
    if bn:
        z = torch.randn(M, cout, device=DEV, generator=g) * 1.5 - 0.3
        mean = -0.3 + 0.1 * torch.randn(cout, device=DEV, generator=g)
        rstd = 0.6 + 0.1 * torch.rand(cout, device=DEV, generator=g)

    def launch():
        if bn:
            o = dict(gy=Out(M * cout), partial=Out(rows * cout * 2))
            rc = L.ga_disc_dgrad(_p(dz), n, H, W, cg, _p(wf), kpf, cout, s, _p(act), _p(z), _p(mean), _p(rstd),
                                 _p(o["gy"].t), _p(o["partial"].t), None, _st())
        else:
            o = dict(out=Out(M * cout, torch.bfloat16))
            rc = L.ga_disc_dgrad(_p(dz), n, H, W, cg, _p(wf), kpf, cout, s, _p(act), None, None, None, None, None,
                                 _p(o["out"].t), _st())
        assert rc == 0
        return o

    o = twice(launch)
    g64, w64 = _nchw(dz), w.to(torch.bfloat16).double()
    mask = _rows(_nchw(act))
    ref = _lrelu(_rows(ref_dgrad(g64, w64, s, H, W)), mask)
    mag = _rows(ref_dgrad(g64.abs(), w64.abs(), s, H, W))
    K = (4 if s == 2 else 16) * cg + 1
    if not bn:
        within(o["out"].t.reshape(M, cout), ref, CF * U * K * mag + BF * ref.abs(), what)
        return
    within(o["gy"].t.reshape(M, cout), ref, CF * U * K * mag, what + " gy")
    part = o["partial"].t.reshape(rows, cout, 2).double()
    assert bool(torch.isfinite(part).all()), "a partial row is not written"
    xhat = (z.double() - mean.double()) * rstd.double()
    K2 = K + 128 + 3
    within(part[..., 0].sum(0), ref.sum(0), CF * U * K2 * mag.sum(0), what + " sum gy")
    within(part[..., 1].sum(0), (ref * xhat).sum(0), CF * U * K2 * (mag * xhat.abs()).sum(0), what + " sum gy xhat")


# ---- ga_disc_bn_backward --------------------------------------------------------------------------------------------
# (what, M, C, rows per partial): BatchNorm 2-4's shapes; the partial rows as the dgrad (128) or conv 5's backward
# (256) would write them
BNB = [("BN2 4x512", 65536, 128, 128), ("BN2 24x24", 144, 128, 128), ("BN3 24x24 n57", 513, 256, 128),
       ("BN3 24x24 n71", 639, 256, 128), ("BN4 24x24", 16, 512, 256), ("BN4 64x64 n9", 441, 512, 256),
       ("BN4 M=2", 2, 512, 256)]


@pytest.mark.parametrize("training", [1, 0], ids=["train", "eval"])
@pytest.mark.parametrize("what,M,Cc,per", BNB, ids=[c[0] for c in BNB])
def test_bn_backward(L, what, M, Cc, per, training):
    """dbeta and dgamma against the fp64 sums of the partials' two halves: |got - ref| <= u |ref| + 2^-52 n sum(|q|)
    (fp32 rounding of an fp64 sum of n terms in another order); k against (S / M, T / M) within the same over M in
    training, exactly (0, 0) in eval.  dz bit for bit against bf16((gamma rstd) ((gy - k.x) - xhat k.y)), xhat =
    (z - mean) rstd, replayed in fp32 numpy from the kernel's k.  With dgamma and dbeta NULL, k and dz keep their
    bits."""
    g = _gen("bnb", what, training)
    nparts = -(-M // per)
    gy = torch.randn(M, Cc, device=DEV, generator=g) * 0.1
    z = torch.randn(M, Cc, device=DEV, generator=g) + 0.2
    mean = 0.2 + 0.05 * torch.randn(Cc, device=DEV, generator=g)
    rstd = 0.8 + 0.2 * torch.rand(Cc, device=DEV, generator=g)
    gamma = 1 + 0.2 * torch.randn(Cc, device=DEV, generator=g)
    # the partials: per block of `per` rows, fp32 (sum gy, sum gy xhat), as the kernels upstream write them
    xh = (z.double() - mean.double()) * rstd.double()
    blk = torch.zeros(nparts * per, Cc, 2, dtype=torch.float64, device=DEV)
    blk[:M, :, 0], blk[:M, :, 1] = gy.double(), gy.double() * xh
    partial = blk.reshape(nparts, per, Cc, 2).sum(1).float().contiguous()

    def launch(grads=True):
        o = dict(k=Out(Cc * 2), dz=Out(M * Cc, torch.bfloat16))
        if grads:
            o.update(dgamma=Out(Cc), dbeta=Out(Cc))
        assert L.ga_disc_bn_backward(_p(gy), _p(z), M, Cc, _p(mean), _p(rstd), _p(gamma), _p(partial), nparts,
                                     training, _p(o["dgamma"].t) if grads else None,
                                     _p(o["dbeta"].t) if grads else None, _p(o["k"].t), _p(o["dz"].t), _st()) == 0
        return o

    o = twice(launch)
    o2 = twice(lambda: launch(False))
    assert torch.equal(_bits(o["k"].t), _bits(o2["k"].t)) and torch.equal(_bits(o["dz"].t), _bits(o2["dz"].t))
    q = partial.double()
    S, T = q[..., 0].sum(0), q[..., 1].sum(0)
    slack = lambda h: 2.0 ** -52 * nparts * q[..., h].abs().sum(0)
    within(o["dbeta"].t, S, U * S.abs() + slack(0), what + " dbeta")
    within(o["dgamma"].t, T, U * T.abs() + slack(1), what + " dgamma")
    k = o["k"].t.reshape(Cc, 2)
    if training:
        within(k[:, 0], S / M, U * (S / M).abs() + slack(0) / M, what + " k.x")
        within(k[:, 1], T / M, U * (T / M).abs() + slack(1) / M, what + " k.y")
    else:
        assert torch.equal(_bits(k), _bits(torch.zeros_like(k)))
    kk = _f32(k)
    gyn, zn, mn, rs, ga = _f32(gy), _f32(z), _f32(mean), _f32(rstd), _f32(gamma)
    xhn = (zn - mn) * rs
    y = (ga * rs) * ((gyn - kk[:, 0]) - xhn * kk[:, 1])
    got = o["dz"].t.view(torch.int16).cpu().numpy().reshape(M, Cc)
    bad = np.argwhere(got != _bf16_bits(y))
    assert bad.size == 0, "%s dz: %d elements differ from the fp32 replay, first %s" % (what, len(bad), bad[0])


# ---- ga_disc_wgrad --------------------------------------------------------------------------------------------------
# (what, n, H, W, Cin, Co, stride, cin_out, splits): H x W the forward's input; splits says how the pixel split falls
WGRAD = [
    ("conv1 24x24", 2, 24, 24, 8, 64, 2, 3, "many"),         # P 288: 2 splits of 160
    ("conv1 27x41", 2, 27, 41, 8, 64, 2, 3, "many"),         # P 520: 3 splits of 192
    ("conv1 64x64", 4, 64, 64, 8, 64, 2, 3, "many"),         # P 4096: 16 splits of 256
    ("conv1 4x512", 4, 512, 512, 8, 64, 2, 3, "empty tail"), # P 262144: 264 splits of 1024, the last 8 empty
    ("conv2 50x70", 4, 25, 35, 64, 128, 2, 64, "many"),      # P 816: 4 splits of 224, the last 144 pixels
    ("conv2 1x512", 1, 256, 256, 64, 128, 2, 64, "empty tail"),  # P 16384: 33 splits of 512, the last empty
    ("conv3 24x24 n57", 57, 6, 6, 128, 256, 2, 128, "many"), # P 513: 3 splits of 192
    ("conv3 64x64", 4, 16, 16, 128, 256, 2, 128, "one"),     # P 256
    ("conv4 24x24", 4, 3, 3, 256, 512, 1, 256, "one"),       # P 16
    ("conv4 64x64 n16", 16, 8, 8, 256, 512, 1, 256, "many"), # P 784: 3 splits of 288
]


def _wgrad_plan(P, Co, Cin):
    """(splits, chunk) as ga_disc_wgrad chooses them from the shapes alone: enough CTAs for two waves of 132 SMs, at
    least 256 pixels a split, chunks rounded up to 32 pixels.  The workspace size checks the split count."""
    tiles = -(-Co // 128) * (16 * Cin // 128)
    s = max(1, min(-(-264 // tiles), -(-P // 256)))
    chunk = -(-(-(-P // s)) // 32) * 32
    return s, chunk


@pytest.mark.parametrize("case", WGRAD, ids=[c[0] for c in WGRAD])
def test_wgrad(L, case):
    """dw against the fp64 weight gradient of the same bf16 operands, channels past cin_out dropped: |got - ref| <=
    2 u K mag, K = chunk + 1 (exact products summed in fp32 over a split's chunk of pixels, the splits in fp64).  The
    workspace is exactly ga_disc_wgrad_workspace_bytes, all of it written."""
    what, n, H, W, cin, co, s, cin_out, kind = case
    g = _gen("wgrad", what)
    Ho, Wo = do.out_size(H, s), do.out_size(W, s)
    P = n * Ho * Wo
    splits, chunk = _wgrad_plan(P, co, cin)
    ws_bytes = L.ga_disc_wgrad_workspace_bytes(n, Ho, Wo, co, cin)
    assert ws_bytes == splits * co * 16 * cin * 4
    assert {"one": splits == 1, "many": splits > 1 and (splits - 1) * chunk < P,
            "empty tail": (splits - 1) * chunk >= P}[kind], (splits, chunk, P)
    dy = torch.randn(n, Ho, Wo, co, device=DEV, generator=g).to(torch.bfloat16)
    x = torch.zeros(n, H, W, cin, device=DEV, dtype=torch.bfloat16)
    x[..., :cin_out] = _act((n, H, W, cin_out), g)         # conv 1: channels 3-7 of the packed image are zero

    def launch():
        o = dict(ws=Out(ws_bytes // 4), dw=Out(co * cin_out * 16))
        assert L.ga_disc_wgrad(_p(dy), _p(x), n, H, W, cin, co, s, cin_out, _p(o["ws"].t), ws_bytes, _p(o["dw"].t),
                               _st()) == 0
        return o

    o = twice(launch)
    assert bool(torch.isfinite(o["ws"].t).all()), "a workspace split is not written"
    g64, x64 = _nchw(dy), _nchw(x[..., :cin_out])
    ref = ref_wgrad(g64, x64, s)
    mag = ref_wgrad(g64.abs(), x64.abs(), s)
    within(o["dw"].t.reshape(co, cin_out, 4, 4), ref, CF * U * (chunk + 1) * mag, what)


# ---- ga_disc_colsum -------------------------------------------------------------------------------------------------
def _colsum_check(L, x, rows, Cc, what):
    """out against the fp64 column sums: |got - ref| <= 2 u K sum(|x|), K = min(rows, 1024) + 1 (a block's fp32 sum,
    the blocks in fp64, one rounding).  Scratch exactly ga_disc_colsum_scratch_bytes, guarded."""
    sb = L.ga_disc_colsum_scratch_bytes(rows, Cc)
    assert sb == -(-rows // 1024) * Cc * 4

    def launch():
        o = dict(scratch=Out(sb // 4), out=Out(Cc))
        assert L.ga_disc_colsum(_p(x), int(x.dtype == torch.bfloat16), rows, Cc, _p(o["scratch"].t), sb,
                                _p(o["out"].t), _st()) == 0
        return o

    o = twice(launch)
    xd = x.double().reshape(rows, Cc)
    within(o["out"].t, xd.sum(0), CF * U * (min(rows, 1024) + 1) * xd.abs().sum(0), what)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("Cc", [1, 2, 64, 256])
def test_colsum(L, Cc, dtype):
    """Row counts around the 1024-row block: 1, 1023, 1024, 1025.  Bound in _colsum_check."""
    for rows in (1, 1023, 1024, 1025):
        g = _gen("colsum", Cc, str(dtype), rows)
        x = (torch.randn(rows, Cc, device=DEV, generator=g) + 0.3).to(dtype)
        _colsum_check(L, x, rows, Cc, "C %d rows %d" % (Cc, rows))


def test_colsum_conv1_bias(L):
    """Conv 1's bias gradient at 16 x 512^2: dz1 bf16 [16 * 256^2, 64].  Bound in _colsum_check."""
    rows = 16 * 256 * 256
    x = (torch.randn(rows, 64, device=DEV, generator=_gen("colsum big")) * 0.01).to(torch.bfloat16)
    _colsum_check(L, x, rows, 64, "conv 1 bias")


# ---- ga_disc_input_backward -----------------------------------------------------------------------------------------
IB = [("24x24", 2, 24, 24), ("27x41", 2, 27, 41), ("50x70", 2, 50, 70), ("64x64", 2, 64, 64), ("4x512", 4, 512, 512),
      ("2x2", 3, 2, 2), ("3x2", 2, 3, 2), ("2x3", 2, 2, 3), ("5x7", 2, 5, 7)]


@pytest.mark.parametrize("what,n,H,W", IB, ids=[c[0] for c in IB])
def test_input_backward(L, what, n, H, W):
    """dx against fp64 conv_transpose of dz1 with the bf16-rounded conv 1 weights the wrapper passes (fp32): |got -
    ref| <= 2 u K mag, K = 4 * 64 + 1 (at most four taps of 64 channels reach a pixel; bf16 x bf16 products are exact
    in fp32)."""
    g = _gen("inb", what)
    Ho, Wo = do.out_size(H, 2), do.out_size(W, 2)
    dz1 = torch.randn(n, Ho, Wo, 64, device=DEV, generator=g).to(torch.bfloat16)
    w1 = torch.randn(64, 3, 4, 4, device=DEV, generator=g) * 0.05
    w1f = w1.to(torch.bfloat16).float().permute(2, 3, 0, 1).reshape(16, 64, 3).contiguous()

    def launch():
        o = Out(n * 3 * H * W)
        assert L.ga_disc_input_backward(_p(dz1), n, H, W, _p(w1f), _p(o.t), _st()) == 0
        return {"dx": o}

    o = twice(launch)["dx"]
    g64, w64 = _nchw(dz1), w1.to(torch.bfloat16).double()
    ref = ref_dgrad(g64, w64, 2, H, W)
    mag = ref_dgrad(g64.abs(), w64.abs(), 2, H, W)
    within(o.t.reshape(n, 3, H, W), ref, CF * U * (4 * 64 + 1) * mag, what)
