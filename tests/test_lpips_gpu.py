"""LPIPS (VGG) and SSIM on the GPU: the ReLU convolution at every VGG layer shape against fp64 with guard bands, the
max pool bit for bit against torch, LPIPS against the bf16-emulating and the fp64 oracle (oracle/lpips_oracle.py) on
the golden inputs, the bit-level properties of the head and the reduction, SSIM against fp64, and the chunk scoring
of gbuffer.py."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import lpips_oracle as lo

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "lpips_small.npz")
CHUNK = os.path.join(ROOT, "tests", "golden", "gbuffer_chunk")
PLY = os.path.join(CHUNK, "fps-4096.ply")
REL_L2 = 6e-3                  # the project's tolerance for bf16 network activations against a bf16-emulating oracle
# LPIPS value, absolute.  Against the bf16-emulating oracle the difference is the GPU's other fp32 summation order
# flipping some bf16 roundings; against fp64 it adds the bf16 bias itself (measured on the CPU up to 8.3e-5 on these
# inputs).  Both bounds sit a few times above the measured differences (see INTEGRATION.md section 3g).
TOL_EMU = 5e-5
TOL_FP64 = 2e-4
SSIM_TOL = 1e-5
GUARD = 0x7F7F                 # bf16 sentinel bits (a finite value the kernels never write)


def _p(t):
    return C.c_void_p(t.data_ptr() if t is not None else 0)


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


@pytest.fixture(scope="module")
def model():
    from gaussiananything_b200 import lpips
    return lpips.LPIPS(state_dict=lo.random_state_dict(0), device=DEV)


def _pack_w(w, cin_p):
    co, ci = w.shape[:2]
    kp = -(-9 * cin_p // 64) * 64
    wp = torch.zeros(co, 3, 3, cin_p)
    wp[..., :ci] = w.permute(0, 2, 3, 1)
    out = torch.zeros(co, kp)
    out[:, :9 * cin_p] = wp.reshape(co, 9 * cin_p)
    return out.to(torch.bfloat16), kp


# (Cin, Cout, H, W): every VGG16 layer shape (the first with its 8-channel packed input), at odd and even sizes
CONV_SHAPES = [(8, 64, 33, 47), (64, 64, 32, 32), (64, 128, 17, 16), (128, 128, 16, 15), (128, 256, 9, 13),
               (256, 256, 8, 8), (256, 512, 7, 9), (512, 512, 5, 7), (512, 512, 4, 4)]


@pytest.mark.parametrize("cin,cout,H,W", CONV_SHAPES)
def test_conv_relu_against_fp64_with_guard_bands(cin, cout, H, W):
    from gaussiananything_b200 import _lib
    L = _lib.lib()
    g = torch.Generator().manual_seed(cin * 7 + cout + H)
    n = 2
    x = torch.randn(n, H, W, cin, generator=g).to(torch.bfloat16)
    w = (torch.randn(cout, cin, 3, 3, generator=g) * (2.0 / (9 * cin)) ** 0.5).to(torch.bfloat16)
    b = torch.randn(cout, generator=g) * 0.05
    wp, kp = _pack_w(w.float(), cin)
    M, pad = n * H * W, 3 * cout + 5
    out = torch.full((M * cout + pad,), GUARD, dtype=torch.int16).view(torch.bfloat16).to(DEV)
    xd, wd, bd = x.to(DEV), wp.to(DEV), b.to(DEV)
    rc = L.ga_conv3x3_relu_bf16(_p(xd), n, H, W, cin, _p(wd), kp, _p(bd), cout, _p(out), _st())
    torch.cuda.synchronize()
    assert rc == 0
    got = out[:M * cout].float().cpu().reshape(n, H, W, cout).permute(0, 3, 1, 2).double()
    assert torch.all(out[M * cout:].view(torch.int16).cpu() == GUARD), "guard band overwritten"
    xc = x.double().permute(0, 3, 1, 2)
    ref = F.conv2d(xc, w.double(), b.double(), padding=1)
    mag = F.conv2d(xc.abs(), w.double().abs(), b.double().abs(), padding=1)
    # bound: half a bf16 ulp of the result plus fp32 accumulation over K = 9 Cin terms
    bound = ref.abs().clamp_min(0) * 2.0 ** -8 + mag * (9 * cin) * 2.0 ** -24 + 1e-30
    err = (got - ref.clamp_min(0)).abs()
    assert float((err / bound).max()) <= 1.0, float((err / bound).max())
    assert torch.all(got >= 0)
    # argument checks are ga_conv3x3_bf16's
    assert L.ga_conv3x3_relu_bf16(_p(xd), n, H, W, cin + 4, _p(wd), kp, _p(bd), cout, _p(out), _st()) == -1
    assert L.ga_conv3x3_relu_bf16(_p(xd), n, H, W, cin, _p(wd), kp, _p(bd), cout + 32, _p(out), _st()) == -1
    assert L.ga_conv3x3_relu_bf16(_p(xd), n, H, W, cin, _p(wd), kp - 64, _p(bd), cout, _p(out), _st()) == -1
    assert L.ga_conv3x3_relu_bf16(_p(xd), n, H, W, cin, _p(wd), kp, _p(bd), cout, None, _st()) == -1


def test_plain_conv_unchanged_and_relu_is_its_clamp():
    from gaussiananything_b200 import _lib
    L = _lib.lib()
    g = torch.Generator().manual_seed(11)
    n, H, W, cin, cout = 2, 19, 21, 64, 128
    x = torch.randn(n, H, W, cin, generator=g).to(torch.bfloat16).to(DEV)
    w = torch.randn(cout, cin, 3, 3, generator=g) * 0.06
    b = (torch.randn(cout, generator=g) * 0.05).to(DEV)
    wp, kp = _pack_w(w.to(torch.bfloat16).float(), cin)
    wp = wp.to(DEV)
    M = n * H * W
    of, ob = torch.empty(M, cout, device=DEV), torch.empty(M, cout, device=DEV, dtype=torch.bfloat16)
    orl = torch.empty(M, cout, device=DEV, dtype=torch.bfloat16)
    assert L.ga_conv3x3_bf16(_p(x), n, H, W, cin, _p(wp), kp, _p(b), cout, 1, None, _p(of), _p(ob), _st()) == 0
    assert L.ga_conv3x3_relu_bf16(_p(x), n, H, W, cin, _p(wp), kp, _p(b), cout, _p(orl), _st()) == 0
    torch.cuda.synchronize()
    assert torch.equal(of.to(torch.bfloat16), ob)
    assert torch.equal(ob.float().clamp_min(0), orl.float())
    ref = F.conv2d(x.double().permute(0, 3, 1, 2).cpu(), w.to(torch.bfloat16).double(), b.double().cpu(), padding=1)
    got = of.double().cpu().reshape(n, H, W, cout).permute(0, 3, 1, 2)
    assert float((got - ref).norm() / ref.norm()) < 1e-5


@pytest.mark.parametrize("H,W,C", [(16, 16, 64), (17, 23, 128), (9, 2, 512), (33, 31, 256)])
def test_maxpool_bit_exact(H, W, C):
    from gaussiananything_b200 import _lib
    x = torch.randn(3, H, W, C, generator=torch.Generator().manual_seed(H * W)).to(torch.bfloat16).to(DEV)
    out = torch.empty(3, H // 2, W // 2, C, device=DEV, dtype=torch.bfloat16)
    assert _lib.lib().ga_maxpool2x2_bf16(_p(x), 3, H, W, C, _p(out), _st()) == 0
    torch.cuda.synchronize()
    want = F.max_pool2d(x.permute(0, 3, 1, 2).float(), 2, 2).to(torch.bfloat16).permute(0, 2, 3, 1)
    assert torch.equal(out.view(torch.int16), want.contiguous().view(torch.int16))


@pytest.mark.parametrize("size", ["64x64", "50x70"])
def test_lpips_against_oracles(model, golden, size):
    sd = lo.random_state_dict(0)
    a, b = torch.from_numpy(golden[size + "/in0"]), torch.from_numpy(golden[size + "/in1"])
    taps, table = model.features(a.to(DEV), b.to(DEV))
    emu = lo.lpips(sd, a, b, emulate_bf16=True)
    f64 = lo.lpips(sd, a, b)
    for k, (t, want) in enumerate(zip(taps, emu["taps"])):
        got = t.double().cpu().permute(0, 3, 1, 2)
        e = float((got - want.double()).norm() / want.double().norm())
        print(size, "tap", k, "rel-L2 vs bf16 oracle", e)
        assert e <= REL_L2, (k, e)
    val = model(a.to(DEV), b.to(DEV)).reshape(-1).double().cpu()
    assert torch.equal(val.float(), table[:, 5].cpu()), "chunked graph path == one eager pass"
    d_emu, d_64 = (val - emu["value"]).abs(), (val - f64["value"]).abs()
    print(size, "lpips", val.tolist(), "|gpu - bf16 oracle|", d_emu.tolist(), "|gpu - fp64|", d_64.tolist())
    assert float(d_emu.max()) <= TOL_EMU and float(d_64.max()) <= TOL_FP64
    per = table[:, :5].double().cpu()
    assert float((per - emu["per_tap"]).abs().max()) <= TOL_EMU


def test_lpips_bit_level_properties(model, golden):
    a = torch.from_numpy(golden["64x64/in0"]).to(DEV)
    b = torch.from_numpy(golden["64x64/in1"]).to(DEV)
    _, per = model(a, a, retPerLayer=True)
    assert torch.all(model(a, a) == 0) and all(torch.all(p == 0) for p in per)
    ab, ba = model(a, b), model(b, a)
    assert torch.equal(ab, ba)
    # one pair alone and the same pair inside 16 (two chunks), at another position
    g = torch.Generator(device=DEV).manual_seed(3)
    big0 = (torch.rand(16, 3, 64, 64, generator=g, device=DEV) * 2 - 1)
    big1 = (torch.rand(16, 3, 64, 64, generator=g, device=DEV) * 2 - 1)
    big0[11], big1[11] = a[2], b[2]
    assert torch.equal(model(big0, big1)[11], model(a[2:3], b[2:3])[0])
    # graph and eager, repeat
    v_graph = model(big0, big1)
    model.use_graph = False
    try:
        v_eager = model(big0, big1)
    finally:
        model.use_graph = True
    assert torch.equal(v_graph, v_eager) and torch.equal(model(big0, big1), v_graph)
    # normalize=True is 2x - 1 first
    assert torch.equal(model((a + 1) / 2, (b + 1) / 2, normalize=True), model(((a + 1) / 2) * 2 - 1, ((b + 1) / 2) * 2 - 1))
    with pytest.raises(RuntimeError, match="inference-only"):
        model(a.clone().requires_grad_(True), b)


def test_ssim_against_fp64(golden):
    from gaussiananything_b200 import lpips
    for size in ("64x64", "50x70"):
        a, b = (torch.from_numpy(golden[size + k]) for k in ("/in0", "/in1"))
        x, y = (a + 1) / 2, (b + 1) / 2
        got = lpips.ssim(x.to(DEV), y.to(DEV)).double().cpu()
        want = lo.ssim(x, y)
        print(size, "ssim", got.tolist(), "|gpu - fp64|", (got - want).abs().tolist())
        assert float((got - want).abs().max()) <= SSIM_TOL
        assert float((got - torch.from_numpy(golden[size + "/ssim"])).abs().max()) <= SSIM_TOL
        assert torch.all(lpips.ssim(x.to(DEV), x.to(DEV)) == 1)
        assert torch.equal(lpips.ssim(x.to(DEV), y.to(DEV)), lpips.ssim(x.to(DEV), y.to(DEV)))
    g = torch.Generator().manual_seed(4)
    x = torch.rand(2, 3, 512, 512, generator=g)
    y = (x + 0.1 * torch.randn(x.shape, generator=g)).clamp(0, 1)
    got = lpips.ssim(x.to(DEV), y.to(DEV)).double().cpu()
    assert float((got - lo.ssim(x, y)).abs().max()) <= SSIM_TOL


def test_perceptual_metrics_of_the_targets_themselves(model):
    from gaussiananything_b200 import gbuffer
    _, t, _ = gbuffer.pack(gbuffer.read_chunk(CHUNK), range(8, 16), DEV)
    same = {"image": ((t["img"] + 1) / 2)[None]}
    m = gbuffer.perceptual_metrics(same, t, model)
    assert m["lpips"].shape == (8,) and m["ssim"].shape == (8,)
    assert torch.all(m["lpips"] == 0) and torch.all(m["ssim"] == 1)
    other = {"image": ((t["img"].roll(1, 0) + 1) / 2)}
    m2 = gbuffer.perceptual_metrics(other, t, model)
    assert torch.all(m2["lpips"] > 0) and torch.all(m2["ssim"] < 1)


def test_reconstruct_chunk_with_and_without_lpips(model):
    from gaussiananything_b200 import vae_decoder as vd
    from gaussiananything_b200 import vae_encoder as ve
    dec = vd.SurfelDecoder(vd.random_state_dict(D=768, depth=2), num_heads=12, depth=2)
    enc = ve.SurfelEncoder(ve.random_state_dict(seed=3), num_frames=8, latent_num=768)
    ae = vd.SurfelAE(dec, encoder=enc)
    run = lambda **kw: ae(behaviour="reconstruct_chunk", chunk=CHUNK, pcd=PLY, fps_start=torch.tensor([5]),
                          generator=torch.Generator().manual_seed(0), **kw)
    plain, scored = run(), run(lpips=model)
    torch.cuda.synchronize()
    for part in ("input", "eval"):
        assert "perceptual" not in plain[part]
        assert set(scored[part]) == set(plain[part]) | {"perceptual"}
        assert torch.equal(scored[part]["table"], plain[part]["table"])
        assert torch.equal(scored[part]["render"]["image"], plain[part]["render"]["image"])
        for k, v in plain[part]["metrics"].items():
            assert torch.equal(scored[part]["metrics"][k], v), k
        p = scored[part]["perceptual"]
        assert p["lpips"].shape == (8,) and p["ssim"].shape == (8,)
        assert torch.all(torch.isfinite(p["lpips"])) and torch.all(p["lpips"] >= 0) and torch.all(p["ssim"] <= 1)
        want = gbuffer_perceptual(scored[part], model)
        assert torch.equal(p["lpips"], want["lpips"]) and torch.equal(p["ssim"], want["ssim"])


def gbuffer_perceptual(part, model):
    from gaussiananything_b200 import gbuffer
    return gbuffer.perceptual_metrics(part["render"], part["targets"], model)
