"""The 3D VAE's own kernels (include/ga_b200.h Part 5 and the VAE decode path of Part 2): ga_conv3x3_bf16,
ga_group_norm_nhwc, ga_heads32_split, ga_micro_attention_bf16 and ga_surfel_cascade_pack, called one by one through
the C ABI and compared element by element with fp64 references computed on the inputs' exact bf16 / fp32 values, at
the encoder's and decoder's shapes and at the tile, chunk and warp edges where the kernels split their work.

The plumbing is tests/test_row_kernels_gpu.py's: every output buffer is followed by a guard tail (NaN, or an int16
sentinel for bf16) that must come back untouched, and every entry point is called twice on the same inputs and must
give the same bits.  Bounds are per element, in the same form: u = 2^-24, mag the expression evaluated on absolute
values, K the length of the longest chain of fp32 roundings behind the element; |got - ref| <= c u K mag, plus
2^-8 |ref| for bf16 results and the documented ulp errors of rsqrtf, __expf, expf, tanhf and log1pf.  A normalised
value carries the error of its rounded fp32 mean, u K mean(|x|) rstd |gamma|, and nothing else from the mean: a group
whose |mean| / std is 1000 is held to a bound that is not looser for the other groups in the same call."""
import pytest
import torch

from tests.test_row_kernels_gpu import (BF, CF, DEV, GUARD16, U, L, Out, _bits, _gen, _p, _randn, _report_worst,  # noqa: F401
                                        _silu, _silu_k, _st, same_bits, twice, within)

pytestmark = pytest.mark.gpu

BADARG = -1


# ---- ga_conv3x3_bf16 ------------------------------------------------------------------------------------------------
def _pack_w(w):
    """w [Cout, Cin, 3, 3] -> bf16 [Cout, k_pitch], column (ky * 3 + kx) * Cin + c, zero past 9 Cin."""
    co, ci = w.shape[:2]
    kp = -(-9 * ci // 64) * 64
    wp = torch.zeros(co, kp, device=DEV, dtype=torch.bfloat16)
    wp[:, :9 * ci] = w.permute(0, 2, 3, 1).reshape(co, 9 * ci)
    return wp, kp


def _conv_rows(x, wp, bias, res, stride, Ho, Wo, rows, chunk=4096):
    """fp64 (ref, S) of output rows `rows` (m = (image, oy, ox)): each row's 9 taps gathered from x bf16 NHWC with the
    padding (stride 1: 1 on every side; stride 2: none on the top / left) as zeros, times the packed weights.
    S = sum |x w| + |bias| + |residual|."""
    n, H, W, Ci = x.shape
    pad = 1 if stride == 1 else 0
    wd = wp[:, :9 * Ci].double().t()
    out, mag = [], []
    for r0 in range(0, rows.numel(), chunk):
        m = rows[r0:r0 + chunk]
        img, p = m // (Ho * Wo), m % (Ho * Wo)
        oy, ox = p // Wo, p % Wo
        taps = []
        for ky in range(3):
            for kx in range(3):
                iy, ix = stride * oy - pad + ky, stride * ox - pad + kx
                ok = (iy >= 0) & (iy < H) & (ix >= 0) & (ix < W)
                v = x[img, iy.clamp(0, H - 1), ix.clamp(0, W - 1)].double()
                taps.append(torch.where(ok[:, None], v, torch.zeros_like(v)))
        A = torch.cat(taps, 1)
        y, s = A @ wd, A.abs() @ wd.abs()
        if bias is not None:
            y, s = y + bias.double(), s + bias.double().abs()
        if res is not None:
            rr = res.reshape(-1, res.shape[-1])[m].double()
            y, s = y + rr, s + rr.abs()
        out.append(y)
        mag.append(s)
    return torch.cat(out), torch.cat(mag)


def _conv_case(Lb, n, H, W, Ci, Co, stride, bias, resid, outs, seed, rows=None, what=""):
    """Runs ga_conv3x3_bf16 twice into guarded buffers and checks `rows` (all when None) against fp64:
    |got - ref| <= u K S (+ 2^-8 |ref| for bf16), K = 9 Cin + 2 (the fp32 accumulation and the bias and residual
    additions), S = sum |x w| + |bias| + |residual|."""
    g = _gen("conv", seed)
    Ho, Wo = Lb.ga_conv3x3_out_size(H, stride), Lb.ga_conv3x3_out_size(W, stride)
    M = n * Ho * Wo
    x = _randn((n, H, W, Ci), g).to(torch.bfloat16)
    wp, kp = _pack_w(_randn((Co, Ci, 3, 3), g, (2.0 / (9 * Ci)) ** 0.5).to(torch.bfloat16))
    b = _randn((Co,), g, 0.3) if bias else None
    res = _randn((M, Co), g) if resid else None

    def launch():
        o = {}
        if "f32" in outs:
            o["f32"] = Out(M * Co)
        if "bf16" in outs:
            o["bf16"] = Out(M * Co, torch.bfloat16)
        assert Lb.ga_conv3x3_bf16(_p(x), n, H, W, Ci, _p(wp), kp, _p(b), Co, stride, _p(res),
                                  _p(o["f32"].t) if "f32" in o else None, _p(o["bf16"].t) if "bf16" in o else None,
                                  _st()) == 0
        return o

    o = twice(launch)
    rows = torch.arange(M, device=DEV) if rows is None else rows
    ref, S = _conv_rows(x, wp, b, res, stride, Ho, Wo, rows)
    e = U * (9 * Ci + 2) * S
    what = "conv3x3 %s" % (what or "n%d %dx%d s%d Cin%d Cout%d" % (n, H, W, stride, Ci, Co))
    if "f32" in o:
        within(o["f32"].t.reshape(M, Co)[rows], ref, e, what + " f32")
    if "bf16" in o:
        within(o["bf16"].t.reshape(M, Co)[rows], ref, e + BF * ref.abs(), what + " bf16")
        if "f32" in o:
            same_bits(o["bf16"].t, o["f32"].t.to(torch.bfloat16), what + " bf16 = bf16(f32)")


# (n, H, W, Cin, Cout, stride, bias, residual, outputs): every Cin and Cout of the sweep, both strides, at stride 2 H and
# W odd, even, 2 and 3; M % 128 of 0, 1 and 127 and M < 128 (n images sharing a 128-row tile)
CONV = [
    (1, 8, 16, 8, 64, 1, True, True, "f32 bf16"),        # M = 128
    (2, 9, 15, 16, 128, 1, False, False, "bf16"),         # M = 270, K % 64 = 16
    (3, 7, 7, 24, 192, 1, True, False, "f32"),           # M = 147 (% 128 = 19), K = 216, three BN = 64 tiles
    (1, 16, 8, 64, 256, 1, False, True, "f32 bf16"),     # M = 128
    (2, 13, 5, 128, 64, 1, True, True, "bf16"),          # M = 130 (% 128 = 2)
    (1, 5, 13, 256, 128, 1, True, False, "f32"),         # M = 65 < 128
    (1, 3, 5, 512, 192, 1, False, False, "f32 bf16"),    # M = 15, K = 4608
    (3, 43, 1, 8, 64, 1, True, True, "f32"),             # M = 129 (% 128 = 1), W = 1
    (1, 127, 1, 16, 256, 1, False, True, "bf16"),        # M = 127
    (2, 16, 16, 64, 64, 2, True, False, "f32"),          # even -> 8 x 8
    (3, 17, 9, 24, 128, 2, True, True, "f32 bf16"),      # odd -> 8 x 4
    (2, 2, 3, 128, 192, 2, False, True, "bf16"),         # 2 x 3 -> 1 x 1
    (3, 3, 2, 256, 256, 2, True, False, "f32"),          # 3 x 2 -> 1 x 1
    (1, 2, 2, 512, 64, 2, True, True, "f32 bf16"),       # 2 x 2 -> 1 x 1
    (2, 33, 20, 8, 128, 2, False, False, "f32"),         # odd / even -> 16 x 10
    (1, 255, 3, 16, 64, 2, True, True, "bf16"),          # 127 x 1: M = 127
    (3, 31, 23, 64, 192, 2, False, True, "f32"),         # 15 x 11: M = 495 (% 128 = 111)
]


@pytest.mark.parametrize("n,H,W,Ci,Co,stride,bias,resid,outs", CONV,
                         ids=["n%d %dx%d Cin%d Cout%d s%d b%d r%d %s" % c for c in CONV])
def test_conv3x3(L, n, H, W, Ci, Co, stride, bias, resid, outs):
    """bias + conv3x3(x) (+ residual) with bias and residual present or NULL, outputs fp32 only, bf16 only or both
    (then bf16 = bf16(fp32) bit for bit).  Bound in _conv_case."""
    _conv_case(L, n, H, W, Ci, Co, stride, bias, resid, outs.split(), ("sweep", n, H, W, Ci, Co, stride))


# the encoder's 3x3 convolutions (ch 64, ch_mult 1 2 4 4) at 2 views of 24 x 20: conv_in, each level's two resnet
# convolutions (the second with the residual, fp32 and bf16) and the three stride-2 downsamples
ENC = [("conv_in", 16, 64, 1, 24, 20, False, "f32"), ("res0.conv1", 64, 64, 1, 24, 20, False, "f32"),
       ("res0.conv2", 64, 64, 1, 24, 20, True, "f32 bf16"), ("down0", 64, 64, 2, 24, 20, False, "f32"),
       ("res1.conv1", 64, 128, 1, 11, 10, False, "f32"), ("res1.conv2", 128, 128, 1, 11, 10, True, "f32 bf16"),
       ("down1", 128, 128, 2, 11, 10, False, "f32"), ("res2.conv1", 128, 256, 1, 5, 5, False, "f32"),
       ("res2.conv2", 256, 256, 1, 5, 5, True, "f32 bf16"), ("down2", 256, 256, 2, 5, 5, False, "f32"),
       ("res3.conv2", 256, 256, 1, 2, 2, True, "f32 bf16")]


@pytest.mark.parametrize("what,Ci,Co,stride,H,W,resid,outs", ENC, ids=[e[0] for e in ENC])
def test_conv3x3_encoder_layers(L, what, Ci, Co, stride, H, W, resid, outs):
    """The encoder's layer shapes at reduced H x W, every output row checked.  Bound in _conv_case."""
    _conv_case(L, 2, H, W, Ci, Co, stride, True, resid, outs.split(), ("enc", what), what="encoder " + what)


def test_conv3x3_lpips_backward_form(L):
    """The LPIPS backward's pooled-map dgrad: Cin 512, Cout 256, no bias, no residual, fp32 only.  Bound in
    _conv_case."""
    _conv_case(L, 2, 13, 11, 512, 256, 1, False, False, ["f32"], ("lpips",), what="lpips dgrad")


def _sampled_rows(M, HoWo, g):
    """The first and last 128-row tiles, the rows on each side of every image boundary and 2048 random rows."""
    edges = [torch.arange(128), torch.arange(M - 128, M)]
    b = torch.arange(1, M // HoWo) * HoWo
    edges += [b - 1, b]
    edges.append(torch.randint(0, M, (2048,), generator=g))
    return torch.unique(torch.cat(edges)).to(DEV)


@pytest.mark.parametrize("what,Ci,Co,stride", [("conv_in", 16, 64, 1), ("down0", 64, 64, 2)], ids=["conv_in", "down0"])
def test_conv3x3_deployed_size(L, what, Ci, Co, stride):
    """B = 2 x 8 views at 512^2: conv_in (16 -> 64) and down.0 (64 -> 64, stride 2) with the encoder's outputs, checked
    at sampled rows (_sampled_rows).  Bound in _conv_case."""
    n, H = 16, 512
    Ho = L.ga_conv3x3_out_size(H, stride)
    rows = _sampled_rows(n * Ho * Ho, Ho * Ho, torch.Generator().manual_seed(7))
    _conv_case(L, n, H, H, Ci, Co, stride, True, False, ["f32"], ("deployed", what), rows=rows,
               what="deployed " + what)


def test_conv3x3_refuses_misaligned_outputs(L):
    """A residual or fp32 output not 8-byte aligned, or a bf16 output not 4-byte aligned, is refused before any launch:
    the call returns GA_ERR_BADARG and the outputs stay untouched."""
    n, H, W, Ci, Co = 1, 4, 4, 8, 64
    x = torch.zeros(n, H, W, Ci, device=DEV, dtype=torch.bfloat16)
    wp, kp = _pack_w(torch.zeros(Co, Ci, 3, 3, device=DEV, dtype=torch.bfloat16))
    M = n * H * W
    res = torch.zeros(M * Co + 2, device=DEV)
    for shift_res, shift_f, shift_b in ((1, 0, 0), (0, 1, 0), (0, 0, 1)):
        of, ob = Out(M * Co + 2), Out(M * Co + 2, torch.bfloat16)
        rc = L.ga_conv3x3_bf16(_p(x), n, H, W, Ci, _p(wp), kp, None, Co, 1, _p(res[shift_res:]), _p(of.t[shift_f:]),
                               _p(ob.t[shift_b:]), _st())
        torch.cuda.synchronize()
        assert rc == BADARG, (shift_res, shift_f, shift_b, rc)
        assert bool(torch.isnan(of.full).all()) and bool((ob.full.view(torch.int16) == GUARD16).all()), \
            "a refused call wrote its outputs"


# ---- ga_group_norm_nhwc ---------------------------------------------------------------------------------------------
RATIOS = (1.0, 100.0, 1000.0, -100.0, -1000.0, 0.3)


def _gn_input(n, HW, Cc, g):
    """x [n, HW, C] whose group k (per image) has std s_k and mean r_k s_k, r_k cycling through RATIOS: groups with
    |mean| / std of 1, 100 and 1000 in the same call."""
    cpg = Cc // 32
    k = torch.arange(32, device=DEV)
    s = 0.5 + 0.25 * (k % 5)
    r = torch.tensor(RATIOS, device=DEV)[k % len(RATIOS)]
    scale = s.repeat_interleave(cpg)
    shift = (r * s).repeat_interleave(cpg)
    return torch.randn((n, HW, Cc), device=DEV, generator=g) * scale + shift


def _gn_check(o, x, gamma, beta, silu, bf16, eps, HW, what):
    """fp64 GroupNorm of x with the group's exact mean and variance.  The fp32 kernel's normalised value t = (x - mean)
    rstd gamma + beta carries 2 u (K |n gamma| + Km mean(|x|) rstd |gamma|) + 2 u |beta|: Km = 4 for the mean rounded
    to fp32 (its fp64 merge adds far less), K = the chunk's per-thread chain (chunk / slots) + slots + the group's
    channels + 16 for the fold, rsqrt, the subtraction and the two products.  SiLU passes that through its slope
    (<= 1.1) and adds __expf's error (_silu_k); a bf16 result adds 2^-8 |ref|."""
    n, _, Cc = x.shape
    cpg = Cc // 32
    cp = 1024 if HW >= 65536 else (256 if HW >= 4096 else 64)
    slots = 256 // (Cc // 4)
    K = -(-cp // slots) + slots + cpg + 16
    xd = x.double().reshape(n, HW, 32, cpg)
    mean = xd.mean((1, 3), keepdim=True)
    var = ((xd - mean) ** 2).mean((1, 3), keepdim=True)
    rs = 1 / (var + eps).sqrt()
    am = xd.abs().mean((1, 3), keepdim=True)
    nrm = ((xd - mean) * rs).reshape(n, HW, Cc)
    gd, bd = gamma.double(), beta.double()
    t = nrm * gd + bd
    gam = gd.abs()
    e = CF * U * (K * (nrm * gd).abs() + 4 * (am * rs).expand(n, 1, 32, cpg).reshape(n, 1, Cc) * gam + bd.abs())
    del xd, nrm
    ref = t
    if silu:
        ref = _silu(t)
        e = 1.1 * e + CF * U * _silu_k(t) * ref.abs()
    if bf16:
        e = e + BF * ref.abs()
    within(o.t.reshape(n, HW, Cc), ref, e, what)
    return float((mean.abs() / var.sqrt()).max())


# (HW, C): every HW of the chunk switch (64 / 256 / 1024 pixels at HW < 4096 / < 65536 / larger) with a full and a
# partial last chunk, every C; silu and the output type alternate
GN = [(1, 32), (63, 1024), (64, 96), (4095, 64), (4096, 512), (65535, 32), (65536, 128), (70000, 256), (4097, 1024),
      (300, 256), (1, 96)]


@pytest.mark.parametrize("out_bf16", [0, 1])
@pytest.mark.parametrize("silu", [0, 1])
@pytest.mark.parametrize("HW,Cc", GN, ids=["HW%d C%d" % c for c in GN])
def test_group_norm(L, HW, Cc, silu, out_bf16):
    """GroupNorm(32) [+ SiLU] -> fp32 or bf16 on 2 images whose groups have |mean| / std of 1, 100 and 1000 side by
    side (_gn_input).  Bound in _gn_check."""
    n, eps = 2, 1e-6
    g = _gen("gn", HW, Cc, silu, out_bf16)
    x = _gn_input(n, HW, Cc, g)
    gamma, beta = _randn((Cc,), g, 0.3, 1.0), _randn((Cc,), g, 0.3)
    nb = L.ga_group_norm_scratch_bytes(n, HW)
    scratch = torch.empty(nb, device=DEV, dtype=torch.uint8)

    def launch():
        o = Out(n * HW * Cc, torch.bfloat16 if out_bf16 else torch.float32)
        assert L.ga_group_norm_nhwc(_p(x), _p(gamma), _p(beta), n, HW, Cc, eps, silu, _p(o.t), out_bf16, _p(scratch),
                                    nb, _st()) == 0
        return {"out": o}

    o = twice(launch)["out"]
    _gn_check(o, x, gamma, beta, silu, out_bf16, eps, HW,
              "group_norm HW%d C%d silu%d %s" % (HW, Cc, silu, "bf16" if out_bf16 else "f32"))


def test_group_norm_deployed_size(L):
    """The encoder's first GroupNorm at B = 2 x 8 views of 512^2: HW 262144, C 64, SiLU, bf16 out.  Bound in
    _gn_check."""
    n, HW, Cc, eps = 16, 512 * 512, 64, 1e-6
    g = _gen("gn deployed")
    x = _gn_input(n, HW, Cc, g)
    gamma, beta = _randn((Cc,), g, 0.3, 1.0), _randn((Cc,), g, 0.3)
    nb = L.ga_group_norm_scratch_bytes(n, HW)
    assert nb == n * (HW // 1024) * 32 * 8
    scratch = torch.empty(nb, device=DEV, dtype=torch.uint8)

    def launch():
        o = Out(n * HW * Cc, torch.bfloat16)
        assert L.ga_group_norm_nhwc(_p(x), _p(gamma), _p(beta), n, HW, Cc, eps, 1, _p(o.t), 1, _p(scratch), nb,
                                    _st()) == 0
        return {"out": o}

    o = twice(launch)["out"]
    for i in range(0, n, 4):                                        # the fp64 reference four images at a time
        sub = Out(4 * HW * Cc, torch.bfloat16)
        sub.t.copy_(o.t[i * HW * Cc:(i + 4) * HW * Cc])
        _gn_check(sub, x[i:i + 4], gamma, beta, 1, 1, eps, HW, "group_norm deployed")


def test_group_norm_refuses(L):
    """x not 16-byte aligned, an fp32 output not 16-byte or a bf16 output not 8-byte aligned, and too little scratch are
    refused before any launch (GA_ERR_BADARG, GA_ERR_WORKSPACE) and the output stays untouched."""
    n, HW, Cc = 1, 64, 64
    x = torch.zeros(n * HW * Cc + 4, device=DEV)
    gamma, beta = torch.ones(Cc, device=DEV), torch.zeros(Cc, device=DEV)
    nb = L.ga_group_norm_scratch_bytes(n, HW)
    scratch = torch.zeros(nb, device=DEV, dtype=torch.uint8)
    for xs, os_, bf16, sb, want in ((1, 0, 0, nb, BADARG), (0, 2, 0, nb, BADARG), (0, 2, 1, nb, BADARG),
                                    (0, 0, 0, nb - 8, -2)):
        o = Out(n * HW * Cc + 4, torch.bfloat16 if bf16 else torch.float32)
        rc = L.ga_group_norm_nhwc(_p(x[xs:]), _p(gamma), _p(beta), n, HW, Cc, 1e-6, 0, _p(o.t[os_:]), bf16,
                                  _p(scratch), sb, _st())
        torch.cuda.synchronize()
        assert rc == want, (xs, os_, bf16, sb, rc)
        untouched = (o.full.view(torch.int16) == GUARD16) if bf16 else torch.isnan(o.full)
        assert bool(untouched.all()), "a refused call wrote its output"


# ---- ga_heads32_split -----------------------------------------------------------------------------------------------
# (B, heads, rows_per_batch, tok_pitch, norm): the SRT's 8 heads over 768 latents at B = 2; rows_per_batch not a
# multiple of 128 with a pitch beyond it; one head; no norm (bit copies)
HEADS = [(2, 8, 768, 768, True), (2, 8, 300, 384, True), (3, 1, 77, 200, True), (2, 8, 129, 256, False),
         (1, 3, 5, 7, True)]


def _heads32_case(Lb, B, Hh, rpb, pitch, norm, key):
    """Runs ga_heads32_split twice into sentinel-filled buffers and checks it (the bound and layout rules of
    test_heads32_split); returns Q, K [B, heads, pitch, 64] and Vt [B, heads, 64, pitch] as written."""
    g = _gen("heads", *key)
    R = B * rpb
    qkv = _randn((R, 3 * Hh * 32), g, 1.5).to(torch.bfloat16)
    qkv[0, :32] = 0                                                 # a zero q row: rsqrt(eps) times zeros
    qn, kn = (_randn((32,), g, 0.3, 1.0), _randn((32,), g, 0.3, 1.0)) if norm else (None, None)
    eps = 1e-5

    def launch():
        o = dict(q=Out(B * Hh * pitch * 64, torch.bfloat16), k=Out(B * Hh * pitch * 64, torch.bfloat16),
                 vt=Out(B * Hh * 64 * pitch, torch.bfloat16))
        assert Lb.ga_heads32_split(_p(qkv), _p(qn), _p(kn), R, Hh, rpb, pitch, eps, _p(o["q"].t), _p(o["k"].t),
                                   _p(o["vt"].t), _st()) == 0
        return o

    o = twice(launch)
    parts = qkv.reshape(B, rpb, 3, Hh, 32).permute(2, 0, 3, 1, 4)          # [3, B, H, rpb, 32]
    for which, w in (("q", qn), ("k", kn)):
        t = o[which].t.reshape(B, Hh, pitch, 64)
        src = parts[0 if which == "q" else 1]
        if w is None:
            same_bits(t[:, :, :rpb, :32], src, "heads32 %s copy" % which)
        else:
            y = src.double()
            ref = y / (y.pow(2).mean(-1, keepdim=True) + eps).sqrt() * w.double()
            within(t[:, :, :rpb, :32], ref, CF * U * 16 * ref.abs() + BF * ref.abs(), "heads32 %s" % which)
        assert bool((_bits(t[:, :, :rpb, 32:]) == 0).all()), "heads32 %s: padding columns not +0" % which
        assert bool((_bits(t[:, :, rpb:]) == GUARD16).all()), "heads32 %s: pitch rows written" % which
    vt = o["vt"].t.reshape(B, Hh, 64, pitch)
    same_bits(vt[:, :, :32, :rpb], parts[2].transpose(-1, -2), "heads32 vt copy")
    assert bool((_bits(vt[:, :, 32:, :rpb]) == 0).all()), "heads32 vt: padding rows not +0"
    assert bool((_bits(vt[..., rpb:]) == GUARD16).all()), "heads32 vt: pitch columns written"
    return o["q"].t.reshape(B, Hh, pitch, 64), o["k"].t.reshape(B, Hh, pitch, 64), vt


@pytest.mark.parametrize("B,Hh,rpb,pitch,norm", HEADS, ids=["B%d H%d rpb%d pitch%d norm%d" % h for h in HEADS])
def test_heads32_split(L, B, Hh, rpb, pitch, norm):
    """q, k = RMSNorm(32)(row) * w -> bf16, against fp64: |got - ref| <= 2 u 16 |ref| + 2^-8 |ref| (the 32-term sum of
    squares by butterfly, rsqrtf's 2 ulp, eps and the two products).  Without weights q and k, and V always, are bit
    copies.  Columns 32..63 of Q and K and rows 32..63 of Vt are +0 for t < rows_per_batch; rows t >= rows_per_batch
    of Q and K and columns t >= rows_per_batch of Vt are the callers' zero fill and stay untouched (sentinels)."""
    _heads32_case(L, B, Hh, rpb, pitch, norm, (B, Hh, rpb, pitch, norm))


def test_heads32_split_feeds_attention(L):
    """The SRT's use: 8 heads of 32 over 300 tokens at B = 2, split (checked as in test_heads32_split), the pitch rows
    zero-filled as the encoder allocates them, then ga_attention_bf16 with scale 32^-0.5 on the padded head_dim 64.
    The attention output is checked element by element against tests/tc_ref.py's fp64 attention of the split's own
    Q, K, Vt (its bound), and columns 32..63 of every head, which only the zero padding of Vt reaches, are 0."""
    from tests import tc_ref
    B, Hh, N, P = 2, 8, 300, 384
    q, k, vt = (t.clone() for t in _heads32_case(L, B, Hh, N, P, True, ("attention", B, Hh, N, P)))
    q[:, :, N:] = 0
    k[:, :, N:] = 0
    vt[..., N:] = 0
    scale = 32 ** -0.5

    def launch():
        o = Out(B * N * Hh * 64, torch.bfloat16)
        assert L.ga_attention_bf16(_p(q), _p(k), _p(vt), _p(o.t), B, Hh, N, N, P, P, scale, 0.0, _st()) == 0
        return {"out": o}

    o = twice(launch)["out"].t.reshape(B, N, Hh, 64)
    ref, tol = tc_ref.attention_ref(q.reshape(B * Hh, P, 64), k.reshape(B * Hh, P, 64), vt.reshape(B * Hh, 64, P), B, Hh,
                                    N, N, scale)
    within(o.reshape(B, N, Hh * 64), ref, tol, "heads32 attention")
    assert float(o[..., 32:].float().abs().max()) == 0.0, "attention columns past head_dim 32 are not 0"


# ---- ga_micro_attention_bf16 ----------------------------------------------------------------------------------------
def _micro_ref(qkv, qn, kn, S, Ln, H, eps):
    """fp64 attention of every (sequence, head) and its bound.  qn = q / rms(q) w_q (likewise k) carries NORM_ARITH =
    2^-16 relative; a score s = qn . kn / 8 then carries e_s = (2 NORM_ARITH + 2 u 72) sum |qn kn| / 8; a probability
    P_ij = softmax_j moves by at most P_ij (e_ij + sum_k P_ik e_ik) with e = e_s + 2 u (2 + 1.16 |s - max|) (__expf) and
    2 u (L + 2) for the fp32 sum and division; O_i = sum_j P_ij v_j adds 2 u L sum_j P_ij |v_j| and 2^-8 |O| for bf16."""
    t = qkv.double().reshape(S, Ln, 3, H, 64).permute(2, 0, 3, 1, 4)      # [3, S, H, L, 64]
    q, k, v = t[0], t[1], t[2]
    qh = q / (q.pow(2).mean(-1, keepdim=True) + eps).sqrt() * qn.double()
    kh = k / (k.pow(2).mean(-1, keepdim=True) + eps).sqrt() * kn.double()
    s = qh @ kh.transpose(-1, -2) / 8
    sa = qh.abs() @ kh.abs().transpose(-1, -2) / 8
    P = torch.softmax(s, -1)
    O = P @ v
    e = (2 * 2.0 ** -16 + CF * U * 72) * sa + CF * U * (2 + 1.16 * (s - s.amax(-1, keepdim=True)).abs() + Ln + 2)
    dP = P * (e + (P * e).sum(-1, keepdim=True))
    va = v.abs()
    bound = dP @ va + CF * U * Ln * (P @ va) + BF * O.abs()
    fold = lambda a: a.permute(0, 2, 1, 3).reshape(S * Ln, H * 64)
    return fold(O), fold(bound), P


def _micro_case(Lb, S, Ln, H, g, what, sharp=False):
    """Runs ga_micro_attention_bf16 twice and checks it (bound in _micro_ref).  Sequence 0's first query is zero (all
    its scores equal), sequence 1's keys are all the same row (every query's scores equal), and in sequence 2 key 0 is
    query 0 (one score dominates); `sharp` norm weights near 3 make every row's scores spread by ~10."""
    Cw = H * 64
    qkv = _randn((S * Ln, 3 * Cw), g, 1.5).to(torch.bfloat16)
    seq = qkv.reshape(S, Ln, 3, H, 64)
    seq[0, 0, 0] = 0
    if S > 1:
        seq[1, :, 1] = seq[1, 0, 1].clone()
    if S > 2:
        seq[2, 0, 1] = seq[2, 0, 0]
    wsc, wsh = (0.3, 3.0) if sharp else (0.3, 1.0)
    qn, kn = _randn((64,), g, wsc, wsh), _randn((64,), g, wsc, wsh)
    eps = 1e-5

    def launch():
        o = Out(S * Ln * Cw, torch.bfloat16)
        assert Lb.ga_micro_attention_bf16(_p(qkv), _p(qn), _p(kn), _p(o.t), S, Ln, H, eps, _st()) == 0
        return {"out": o}

    o = twice(launch)["out"]
    ref, bound, P = _micro_ref(qkv, qn, kn, S, Ln, H, eps)
    within(o.t.reshape(S * Ln, Cw), ref, bound, "micro_attention " + what)
    if S > 2 and Ln > 1:
        assert float(P[2, :, 0, 0].min()) > 0.9, "the dominant score does not dominate"
    return P


MICRO = [(Ln, H) for Ln in range(1, 17) for H in (1, 12)]


@pytest.mark.parametrize("Ln,H", MICRO, ids=["L%d H%d" % m for m in MICRO])
def test_micro_attention(L, Ln, H):
    """Every L from 1 to 16 (4, 5 and 9 take the small kernels, the others the generic one) with one head, where S H
    % 4 cycles through 1, 2 and 3 so the last CTA's 4 warps are partly idle, and with the decoder's 12 heads.  Bound
    in _micro_ref; special rows in _micro_case."""
    S = 37 + Ln % 3 if H == 1 else 5
    _micro_case(L, S, Ln, H, _gen("micro", Ln, H), "L%d H%d S%d" % (Ln, H, S), sharp=Ln % 2 == 1)


@pytest.mark.parametrize("S,Ln", [(768, 9), (6144, 5), (24576, 4)], ids=["stage1", "stage2", "stage3"])
def test_micro_attention_deployed(L, S, Ln):
    """The decoder's three up-sampling stages at B = 1: 12 heads over (S, L) = (768, 9), (6144, 5), (24576, 4).  Bound
    in _micro_ref."""
    _micro_case(L, S, Ln, 12, _gen("micro deployed", S, Ln), "deployed S%d L%d" % (S, Ln))


def test_micro_attention_refuses_misaligned(L):
    """qkv or out not 4-byte aligned, qn_w or kn_w not 8-byte aligned: GA_ERR_BADARG before any launch, out untouched."""
    S, Ln, H = 2, 4, 1
    qkv = torch.zeros(S * Ln * 3 * 64 + 2, device=DEV, dtype=torch.bfloat16)
    w = torch.ones(66, device=DEV)
    for qs, os_, qw, kw in ((1, 0, 0, 0), (0, 1, 0, 0), (0, 0, 1, 0), (0, 0, 0, 1)):
        o = Out(S * Ln * 64 + 2, torch.bfloat16)
        rc = L.ga_micro_attention_bf16(_p(qkv[qs:]), _p(w[qw:]), _p(w[kw:]), _p(o.t[os_:]), S, Ln, H, 1e-5, _st())
        torch.cuda.synchronize()
        assert rc == BADARG, (qs, os_, qw, kw, rc)
        assert bool((o.full.view(torch.int16) == GUARD16).all()), "a refused call wrote its output"


# ---- ga_surfel_cascade_pack -----------------------------------------------------------------------------------------
def _pack_ref(res, pre, parent_pos_rows, offset_scale, sf, parent_pre):
    """oracle/vae_decoder_oracle.Activations in float64: xyz = tanh(res[0:3]) offset_scale + parent_pos, then sigmoid |
    softplus (threshold 20) * sf | F.normalize | 0.5 tanh + 0.5 of pre; and the per-channel bound 2 u (K mag):
    tanhf 2 ulp + product + sum on the position; the fp32 pre = res + parent_pre rounding (u |pre|, through slopes <=
    1) on the others plus expf / log1pf / tanhf's ulps, the sum of squares, sqrtf and the division."""
    from oracle import vae_decoder_oracle as vo
    act = vo.Activations(0.45)
    act.scaling_factor = torch.tensor(sf, dtype=torch.float64)
    r, p = res.double(), pre.double()
    th = torch.tanh(r[:, :3])
    pos = th * offset_scale + parent_pos_rows.double()
    ref = act.pack(pos, p)
    pe = p.abs() if parent_pre else torch.zeros_like(p)
    e = torch.empty_like(ref)
    e[:, :3] = 4 * (th * offset_scale).abs() + ref[:, :3].abs()
    e[:, 3] = 6 * ref[:, 3].abs() + 0.25 * pe[:, 3]
    e[:, 4:6] = (4 * ref[:, 4:6].abs() / sf + 4 + pe[:, 4:6]) * sf
    e[:, 6:10] = 10 * ref[:, 6:10].abs() + 2 * pe[:, 6:10] / p[:, 6:10].norm(dim=-1, keepdim=True).clamp_min(1e-12)
    e[:, 10:] = 4 * (0.5 * torch.tanh(p[:, 10:])).abs() + 2 * ref[:, 10:].abs() + 0.5 * pe[:, 10:]
    return ref, CF * U * e


# (N parents, f, res_in_sequences, out_pre): the base level (f 1, parent_pre NULL, parent_pos stride 3); the cascade's
# child levels f 8, 4, 3 with the parent's 13-wide gaussians as positions; R = N f never a multiple of 256
PACK = [(301, 1, 0, 1), (301, 1, 0, 0), (37, 8, 0, 1), (37, 8, 1, 0), (101, 4, 1, 1), (101, 4, 0, 0), (95, 3, 1, 1),
        (95, 3, 0, 1)]


def _pack_level(Lb, res, in_seq, parent_pre, ppos, f, with_pre, what):
    """Runs ga_surfel_cascade_pack twice on res [R, 13] (laid out in [N, 1 + f] sequences with NaN parent rows when
    in_seq), parent_pre [N, 13] or None (the base level) and the parents' positions ppos [N, stride], and checks it
    against Activations in float64 (bound in _pack_ref); out_pre = res + parent_pre bit for bit (fp32, one rounding).
    Returns (gaussians [R, 13], pre [R, 13]) as the next level takes them."""
    from oracle import vae_decoder_oracle as vo
    base = parent_pre is None
    R, N, stride = res.shape[0], ppos.shape[0], ppos.shape[1]
    if in_seq:
        res_arg = torch.full((N, 1 + f, 13), float("nan"), device=DEV)
        res_arg[:, 1:] = res.reshape(N, f, 13)
    else:
        res_arg = res
    f32 = lambda v: float(torch.tensor(float(v), dtype=torch.float32))   # the values the kernel gets
    os_, sf = f32(0.45 * 0.5 * (0.1 if base else 1.0)), f32(vo.Activations(0.45).scaling_factor)

    def launch():
        o = {"g": Out(R * 13)}
        if with_pre:
            o["pre"] = Out(R * 13)
        assert Lb.ga_surfel_cascade_pack(_p(res_arg), in_seq, _p(parent_pre), _p(ppos), stride, f, os_, sf,
                                         _p(o["g"].t), _p(o["pre"].t) if with_pre else None, R, _st()) == 0
        return o

    o = twice(launch)
    pi = torch.arange(R, device=DEV) // f
    pre = res if base else res + parent_pre[pi]
    ref, bound = _pack_ref(res, pre, ppos[pi, :3], os_, sf, not base)
    got = o["g"].t.reshape(R, 13)
    within(got, ref, bound, "surfel_pack " + what)
    if with_pre:
        same_bits(o["pre"].t.reshape(R, 13), pre, "surfel_pack pre " + what)
    return got, pre


@pytest.mark.parametrize("N,f,in_seq,with_pre", PACK, ids=["N%d f%d seq%d pre%d" % p for p in PACK])
def test_surfel_cascade_pack(L, N, f, in_seq, with_pre):
    """One level (checks in _pack_level).  Channels 4-5 of the first rows are 20 and 20 +- 1 ulp (softplus's
    threshold), and some rows have a zero quaternion (F.normalize gives +0, not NaN).  The sequence layout's parent
    rows and the position rows' channels 3..12 are NaN: the kernel must not read them."""
    g = _gen("pack", N, f, in_seq, with_pre)
    base = f == 1
    R = N * f
    res = _randn((R, 13), g, 2.0)
    if base:
        t20 = torch.tensor([20.0], device=DEV)
        near = torch.cat([torch.nextafter(t20, t20 - 1), t20, torch.nextafter(t20, t20 + 1)])
        res[:3, 4] = near
        res[:3, 5] = near.flip(0)
        res[3:5, 6:10] = 0
    parent_pre = None if base else _randn((N, 13), g, 2.0)
    if not base:
        parent_pre[1, 6:10] = 0
        res[f:2 * f, 6:10] = 0                                      # pre of parent 1's children: a zero quaternion
    ppos = _randn((N, 3 if base else 13), g, 0.3)
    if not base:
        ppos[:, 3:] = float("nan")
    got, pre = _pack_level(L, res, in_seq, parent_pre, ppos, f, with_pre, "N%d f%d" % (N, f))
    zq = (pre[:, 6:10] == 0).all(-1)
    assert bool(zq.any()) and bool((_bits(got[zq, 6:10]) == 0).all()), "a zero quaternion does not give +0"


def test_surfel_cascade_pack_chain(L):
    """The decoder's cascade as it chains the levels: the base level of 37 tokens, then f = 8, 4 and 3, each level
    taking the previous level's kernel outputs as parent_pre (its out_pre) and parent positions (its 13-wide
    gaussians, stride 13), the residuals alternately in row and sequence layout.  Each level is checked against
    Activations in float64 on its actual inputs (_pack_level); the last level has 37 * 96 surfels."""
    g = _gen("pack chain")
    N = 37
    gs, pre = _pack_level(L, _randn((N, 13), g, 2.0), 0, None, _randn((N, 3), g, 0.3), 1, True, "chain base")
    for i, f in enumerate((8, 4, 3)):
        gs, pre = _pack_level(L, _randn((N * f, 13), g, 2.0), i % 2, pre, gs, f, True, "chain f%d" % f)
        N *= f
    assert N == 37 * 96 and bool(torch.isfinite(gs).all())
