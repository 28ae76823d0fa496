"""The DINOv2 image conditioner (SURVEY.md 8f row N3) on the GPU: the front-end kernel against the oracle's
preprocess, the attention kernel at the encoder's shape, the encoder against the bf16-emulating and fp32 oracles,
the embedder / conditioner interfaces, and image -> conditioner -> DiT-L end to end."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

N_TOK, PITCH, K_PITCH = 1374, 1408, 640


def rel(a, b):
    return float((a.double().cpu() - b.double().cpu()).norm() / b.double().cpu().norm().clamp_min(1e-30))


def _img(B, H, W, seed, device="cpu"):
    return (torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(seed)) * 2 - 1).to(device)


def _env():
    from gaussiananything_b200 import _lib, dit
    dev = torch.device("cuda:0")
    return dit, _lib.lib(), dev, C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _bf16_ulp(x):
    e = torch.floor(torch.log2(x.abs().clamp_min(1e-30)))
    return torch.exp2(e - 7)


@pytest.mark.parametrize("H,W", [(518, 518), (256, 256), (1024, 1024), (700, 400)])
def test_frontend_patch_matrix_matches_oracle(H, W):
    """518^2 (identity resize): bit-exact.  Upscale, blur + downscale, anisotropic: within one bf16 ulp of the
    oracle's fp32 value rounded to bf16, plus 1e-6 absolute: the kernel and torch's CPU bicubic sum the same fp32 taps in
    a different order (and with or without FMA), a few fp32 ulps apart, and where (x - mean) cancels to near zero
    that difference is larger than a bf16 ulp of the result.  Columns 588..639 are zero."""
    from oracle import dino_oracle as do
    dit, L, dev, st = _env()
    B = 2
    img = _img(B, H, W, H * 7 + W)
    nbytes = int(L.ga_dino_frontend_scratch_bytes(B, H, W, 518))
    assert (nbytes > 0) == (H > 518 or W > 518)
    scratch = torch.empty(max(nbytes, 1), device=dev, dtype=torch.uint8)
    out = torch.full((B * 1369, K_PITCH), float("nan"), device=dev, dtype=torch.bfloat16)
    x = img.to(dev)
    rc = L.ga_dino_frontend(dit._p(x), B, H, W, 518, 14, dit._p(out), K_PITCH, dit._p(scratch), nbytes, st)
    assert rc == 0, rc
    torch.cuda.synchronize()
    got = out.float().cpu()
    assert float(got[:, 588:].abs().max()) == 0.0
    want = do.patch_matrix(do.preprocess(img)).bfloat16().float()
    if (H, W) == (518, 518):
        assert torch.equal(got, want)
    else:
        d = (got - want).abs()
        ulp = _bf16_ulp(torch.maximum(got.abs(), want.abs()))
        assert bool((d <= ulp + 1e-6).all()), float((d - ulp).max())
        assert float((d == 0).float().mean()) > 0.99
        assert rel(got, want) < 2e-3


def test_frontend_rejects_bad_sizes():
    """Argument checks that return before any launch."""
    dit, L, dev, st = _env()
    x = torch.zeros(1, 3, 64, 64, device=dev)
    out = torch.zeros(1369, K_PITCH, device=dev, dtype=torch.bfloat16)
    assert L.ga_dino_frontend(dit._p(x), 1, 64, 64, 520, 14, dit._p(out), K_PITCH, None, 0, st) == -1     # not 14 k
    assert L.ga_dino_frontend(dit._p(x), 1, 64, 64, 518, 14, dit._p(out), 584, None, 0, st) == -1         # < 588
    assert L.ga_dino_frontend(dit._p(x), 1, 4100, 64, 518, 14, dit._p(out), K_PITCH, None, 0, st) == -3   # > 4096
    assert L.ga_dino_frontend(dit._p(x), 1, 1024, 64, 518, 14, dit._p(out), K_PITCH, None, 0, st) == -2   # no scratch
    assert L.ga_dino_frontend_scratch_bytes(1, 1024, 64, 518) == 2 * 3 * 1024 * 64 * 4


def test_attention_at_encoder_shape():
    """B = 2, 16 heads, Nq = Nk = 1374 tokens at pitch 1408, no score bound (online softmax), against SDPA."""
    dit, L, dev, st = _env()
    torch.manual_seed(11)
    B, H, N = 2, 16, N_TOK
    q = torch.zeros(B * H, PITCH, 64, device=dev, dtype=torch.bfloat16)
    k = torch.zeros(B * H, PITCH, 64, device=dev, dtype=torch.bfloat16)
    vt = torch.zeros(B * H, 64, PITCH, device=dev, dtype=torch.bfloat16)
    q[:, :N] = torch.randn(B * H, N, 64, device=dev) * 1.2
    k[:, :N] = torch.randn(B * H, N, 64, device=dev) * 1.2
    vt[:, :, :N] = torch.randn(B * H, 64, N, device=dev)
    out = torch.zeros(B, N, H * 64, device=dev, dtype=torch.bfloat16)
    rc = L.ga_attention_bf16(dit._p(q), dit._p(k), dit._p(vt), dit._p(out), B, H, N, N, PITCH, PITCH, 0.125, 0.0, st)
    assert rc == 0, rc
    torch.cuda.synchronize()
    ref = torch.nn.functional.scaled_dot_product_attention(
        q[:, :N].float().view(B, H, N, 64), k[:, :N].float().view(B, H, N, 64),
        vt[:, :, :N].float().transpose(-1, -2).reshape(B, H, N, 64))
    ref = ref.transpose(1, 2).reshape(B, N, H * 64)
    assert rel(out.float(), ref) < 6e-3, rel(out.float(), ref)


def test_encoder_depth4_every_block_matches_emulating_oracle():
    from gaussiananything_b200 import dino
    from oracle import dino_oracle as do
    sd = dino.random_state_dict(4, seed=2)
    enc = dino.Dinov2Encoder(sd, "cuda:0")
    img = _img(2, 518, 518, 21)
    out = enc.encode(img.cuda(), return_acts=True)
    want = do.forward(sd, img, emulate_bf16=True, return_acts=True)
    errs = {"block%d" % i: rel(a, b) for i, (a, b) in enumerate(zip(out["acts"], want["acts"]))}
    errs.update({k: rel(out[k], want[k]) for k in ("x_norm_clstoken", "x_norm_patchtokens")})
    assert len(out["acts"]) == 4 and out["acts"][0].shape == (2, N_TOK, 1024)
    assert all(e <= 6e-3 for e in errs.values()), errs


@pytest.fixture(scope="module")
def deep():
    from gaussiananything_b200 import dino
    sd = dino.random_state_dict(24, seed=0)
    return sd, dino.Dinov2Encoder(sd, "cuda:0")


def test_encoder_depth24_against_oracles_batch_and_graph(deep):
    from oracle import dino_oracle as do
    sd, enc = deep
    img = _img(2, 518, 518, 5)
    enc.use_graph = False
    eager = enc.encode(img.cuda())
    enc.use_graph = True
    g1 = enc.encode(img.cuda())
    g2 = enc.encode(img.cuda())
    assert eager["x_norm_patchtokens"].shape == (2, 1369, 1024) and eager["x_norm_clstoken"].shape == (2, 1024)
    for k in ("x_norm_clstoken", "x_norm_patchtokens"):
        assert torch.isfinite(g1[k]).all(), k
        assert torch.equal(g1[k], eager[k]) and torch.equal(g2[k], g1[k]), k
    emu = do.forward(sd, img, emulate_bf16=True)
    f32 = do.forward(sd, img)
    errs = {k: (rel(g1[k], emu[k]), rel(g1[k], f32[k])) for k in ("x_norm_clstoken", "x_norm_patchtokens")}
    assert all(a <= 6e-3 and b <= 2e-2 for a, b in errs.values()), errs
    one = enc.encode(img[1:].cuda())
    for k in ("x_norm_clstoken", "x_norm_patchtokens"):
        assert rel(one[k][0], g1[k][1]) <= 1e-6, k


def test_embedder_interface(deep):
    from gaussiananything_b200 import dino
    sd, enc = deep
    emb = dino.FrozenDinov2ImageEmbedder(arch="vitl", inp_size=518, output_cls=True, encoder=enc)
    img = _img(1, 518, 518, 8, "cuda").bfloat16()
    out = emb(img)
    assert isinstance(out, tuple) and len(out) == 2
    tokens, z = out
    assert tokens.shape == (1, 1369, 1024) and z.shape == (1, 1024)
    assert tokens.dtype == torch.bfloat16 and z.dtype == torch.bfloat16
    ref = enc.encode(img)
    assert torch.equal(tokens, ref["x_norm_patchtokens"].bfloat16()) and torch.equal(z, ref["x_norm_clstoken"].bfloat16())


class _Counting:
    def __init__(self, enc):
        self.enc, self.calls = enc, 0

    def encode(self, img, **kw):
        self.calls += 1
        return self.enc.encode(img, **kw)


def _conditioners(enc):
    from gaussiananything_b200 import dino
    cnt = _Counting(enc)
    emb = dino.FrozenDinov2ImageEmbedder(arch="vitl", inp_size=518, output_cls=True, encoder=cnt)
    emb.input_key = "img"
    c1 = dino.GeneralConditioner([emb])
    c2 = dino.GeneralConditioner([emb, {"input_key": "fps-xyz", "ucg_rate": 0.0,
                                        "target": "sgm.modules.encoders.modules.PCD_Scaler",
                                        "params": {"scaling_factor": 0.45}}])
    return cnt, c1, c2


def test_conditioner_stage_rules_on_gpu(deep):
    sd, enc = deep
    cnt, c1, c2 = _conditioners(enc)
    img = _img(1, 640, 480, 9, "cuda")
    c, uc = c1.get_unconditional_conditioning({"img": img}, force_uc_zero_embeddings=["img"])
    assert cnt.calls == 1
    assert float(uc["img_crossattn"].abs().max()) == 0 and float(uc["img_vector"].abs().max()) == 0
    assert float(c["img_crossattn"].abs().max()) > 0 and float(c["img_vector"].abs().max()) > 0
    xyz = torch.rand(1, 768, 3, device="cuda") * 0.9 - 0.45
    c, uc = c2.get_unconditional_conditioning({"img": img, "fps-xyz": xyz}, force_uc_zero_embeddings=["img-xyz"])
    assert cnt.calls == 2
    assert sorted(c) == ["fps-xyz", "img_crossattn", "img_vector"] and all(torch.equal(c[k], uc[k]) for k in c)
    assert torch.equal(c["fps-xyz"], xyz / 0.45)


def test_image_to_dit_end_to_end(deep):
    """image -> conditioner -> one forward_with_cfg of a random-init stage-1 DiT-L at N = 768: finite, and the same
    bits as the DiT fed the same context tensors directly."""
    from gaussiananything_b200 import dit
    sd, enc = deep
    cnt, c1, _ = _conditioners(enc)
    img = _img(1, 518, 518, 10, "cuda")
    c, uc = c1.get_unconditional_conditioning({"img": img}, force_uc_zero_embeddings=["img"])
    ctx = {k: torch.cat([c[k], uc[k]], 0) for k in ("img_crossattn", "img_vector")}
    torch.manual_seed(4)
    m = dit.DiT_models["DiT-PixArt-PCD-CLAY-L"](input_size=32, num_classes=0, learn_sigma=False, in_channels=3,
                                                context_dim=1024, roll_out=True, pooling_ctx_dim=768)
    m.randomize_zero_init_().cuda().eval()
    x = torch.randn(1, 768, 3, device="cuda").repeat(2, 1, 1)
    t = torch.full((2,), 0.4, device="cuda")
    with torch.no_grad():
        y = m.forward_with_cfg(x, t, ctx, 4.0)
        y_direct = m.forward_with_cfg(x, t, {k: v.clone() for k, v in ctx.items()}, 4.0)
    assert torch.isfinite(y).all() and float(y.abs().mean()) > 0
    assert torch.equal(y, y_direct)
