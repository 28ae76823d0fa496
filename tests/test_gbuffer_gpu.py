"""G-buffer chunk front end on the GPU: ga_gbuffer_pack and ga_recon_metrics against oracle/gbuffer_oracle.py on the
committed chunk, the encoder on a real (structured) input against its bf16-emulating oracle, and the whole
'reconstruct_chunk' behaviour with random weights."""
import ctypes as C
import os

import pytest
import torch

from oracle import gbuffer_oracle as go
from oracle import vae_encoder_oracle as vo

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHUNK = os.path.join(ROOT, "tests", "golden", "gbuffer_chunk")
PLY = os.path.join(CHUNK, "fps-4096.ply")
# Rays and xyz against the fp64 oracle: 1e-6 absolute.  The largest magnitudes are |o x d| < 1.6 (fp32 spacing 1.2e-7)
# and each value is about ten fp32 roundings deep, so this is the rounding scale, not a tuned number.
RAY_TOL = 1e-6


def _p(t):
    return C.c_void_p(t.data_ptr() if t is not None else 0)


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.fixture(scope="module")
def chunk():
    from gaussiananything_b200 import gbuffer
    return gbuffer.read_chunk(CHUNK)


def _check_pack(enc, t, want):
    e, w = enc.double().cpu(), want["img_to_encoder"]
    assert torch.equal(e[:, :6], w[:, :6]), "rgb / normal channels are the fp32 formula bit for bit"
    assert float((e[:, 6:12] - w[:, 6:12]).abs().max()) <= RAY_TOL
    # xyz: the same zero set, except where the fp64 coordinate is within RAY_TOL of the clip value
    o, d = go.sampler_rays(want["c"].numpy(), 512)
    raw = (o[:, None, :] + want["depth"].double().reshape(len(o), -1, 1) * d).reshape(len(o), 512, 512, 3).permute(0, 3, 1, 2)
    band = (raw.abs() - go.XYZ_CLIP).abs() <= RAY_TOL
    assert float(band.double().mean()) < 1e-4
    assert torch.equal((e[:, 12:] == 0) | band, (w[:, 12:] == 0) | band)
    assert float(((e[:, 12:] - w[:, 12:]).abs() * (~band)).max()) <= RAY_TOL
    if t is not None:
        for k in ("img", "alpha", "depth", "mask"):
            assert torch.equal(t[k].cpu(), want[k]), k
        assert t["normal"].data_ptr() == enc[:, 3:6].data_ptr()


def test_pack_all_views_against_oracle(chunk):
    from gaussiananything_b200 import gbuffer
    enc, t, c = gbuffer.pack(chunk, None, DEV)
    torch.cuda.synchronize()
    assert tuple(enc.shape) == (16, 15, 512, 512) and torch.equal(c.cpu(), torch.from_numpy(chunk["c"]))
    _check_pack(enc, t, go.pack(chunk, None, torch.float64))
    # from device-resident inputs, without targets: the same encoder input
    enc2, t2, _ = gbuffer.pack(gbuffer.to_device(chunk, DEV), None, DEV, with_targets=False)
    assert t2 is None and torch.equal(enc, enc2)


def test_pack_view_subset_leaves_other_rows_alone(chunk):
    from gaussiananything_b200 import _lib, gbuffer
    views = [11, 0, 6, 6, 13]
    V = len(views)
    d = gbuffer.to_device(chunk, DEV)
    vi = torch.tensor(views, dtype=torch.int32, device=DEV)
    GUARD = -777.0
    enc = torch.full((V + 1, 15, 512, 512), GUARD, device=DEV)
    outs = [torch.full((V + 1, ch, 512, 512), GUARD, device=DEV) for ch in (3, 1, 1, 1)]
    rc = _lib.lib().ga_gbuffer_pack(_p(d["raw_img"]), _p(d["normal"]), _p(d["alpha"]), _p(d["depth"]), _p(d["c"]), 16, 512,
                                    512, _p(vi), V, _p(enc), *[_p(o) for o in outs], _st())
    torch.cuda.synchronize()
    assert rc == 0
    assert float(enc[V].min()) == GUARD == float(enc[V].max())
    assert all(float(o[V].min()) == GUARD == float(o[V].max()) for o in outs)
    t = dict(zip(("img", "alpha", "depth", "mask"), (o[:V] for o in outs)), normal=enc[:V, 3:6])
    _check_pack(enc[:V], t, go.pack(chunk, views, torch.float64))
    assert torch.equal(enc[2], enc[3])
    # argument checks return before any launch
    L = _lib.lib()
    bad = lambda **kw: L.ga_gbuffer_pack(*[kw.get(k, v) for k, v in (
        ("raw", _p(d["raw_img"])), ("normal", _p(d["normal"])), ("alpha", _p(d["alpha"])), ("depth", _p(d["depth"])),
        ("c", _p(d["c"])), ("n", 16), ("H", 512), ("W", 512), ("views", _p(vi)), ("V", V), ("enc", _p(enc)),
        ("t0", _p(outs[0])), ("t1", _p(outs[1])), ("t2", _p(outs[2])), ("t3", _p(outs[3])), ("st", _st()))])
    assert bad(raw=None) == -1 and bad(W=510) == -1 and bad(V=0) == -1 and bad(t2=None) == -1 and bad(alpha=None) == -1
    torch.cuda.synchronize()


def _targets(chunk, views):
    from gaussiananything_b200 import gbuffer
    _, t, _ = gbuffer.pack(chunk, views, DEV)
    return t


def _near(t, noise, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    r = lambda ref: torch.rand(ref.shape, generator=g, device=DEV) - 0.5
    return {"image": ((t["img"] + 1) / 2 + noise * r(t["img"])).clamp(0, 1)[None],
            "depth": (t["depth"] + noise * r(t["depth"]))[None],
            "alpha": (t["alpha"] + noise * r(t["alpha"])).clamp(0, 1)[None],
            "rend_normal": torch.nn.functional.normalize(t["normal"] + noise * r(t["normal"]), dim=1)[None]}


def test_metrics_against_oracle_and_bitwise_repeatable(chunk):
    from gaussiananything_b200 import gbuffer
    t = _targets(chunk, [8, 3, 14])
    for k in ("alpha", "depth", "mask"):                                            # view 1: all background
        t[k][1] = 0
    r = _near(t, 0.2, 1)
    tab = gbuffer.metric_table(r, t)
    tab2 = gbuffer.metric_table(r, t)
    torch.cuda.synchronize()
    assert torch.equal(tab, tab2), "two runs give the same bits"
    want = go.metric_table({k: v[0] for k, v in r.items()}, t)
    rel = ((tab.double().cpu() - want).abs() / want.abs().clamp_min(1e-30))
    rel[want == 0] = (tab.double().cpu()[want == 0]).abs()
    assert float(rel.max()) <= 1e-5, rel
    m = gbuffer.derive(tab)
    assert all(torch.isfinite(v).all() for v in m.values())
    assert float(m["fg_pixels"][1]) == 0 and float(m["depth_l1"][1]) == 0 and float(m["normal_error"][1]) == 0
    assert float(tab[0, 7]) == 512 * 512 and float(tab[0, 2]) == float(t["mask"][0].sum())


def test_metrics_of_the_targets_themselves(chunk):
    """The targets as the prediction: capped PSNR, zero depth and alpha error, IoU 1.  The normal error is what the
    8-bit normals leave, 1 - |n|^2 averaged over the foreground (they are not unit length), and equals the oracle's."""
    from gaussiananything_b200 import gbuffer
    t = _targets(chunk, range(8, 16))
    same = {"image": (t["img"] + 1) / 2, "depth": t["depth"], "alpha": t["alpha"], "rend_normal": t["normal"].contiguous()}
    tab = gbuffer.metric_table(same, t)
    m = gbuffer.derive(tab)
    assert torch.all(m["psnr"] == gbuffer.PSNR_CAP) and torch.all(m["depth_l1"] == 0) and torch.all(m["alpha_l1"] == 0)
    assert torch.all(m["iou"] == 1)
    want = go.derive(go.metric_table(same, t))["normal_error"]
    assert float((m["normal_error"] - want).abs().max()) < 1e-6 and float(m["normal_error"].abs().max()) < 0.02


def test_encoder_on_a_real_input_against_bf16_oracle(chunk):
    """The encoder's first structured input (clipped xyz with zeroed background, unit rays, moments, normals): two
    views of the chunk at every 8th pixel (64 x 64), the first 512 surface samples, 64 latents -- the sizes and the
    tolerance of tests/test_vae_encoder_gpu.py::test_encoder_against_bf16_oracle, whose input is randn."""
    from gaussiananything_b200 import gbuffer
    from gaussiananything_b200 import vae_encoder as ve
    V, K = 2, 64
    enc_in, _, _ = gbuffer.pack(chunk, [1, 9], DEV, with_targets=False)
    img = enc_in[:, :, 4::8, 4::8].contiguous()
    assert float((img[:, 12:] == 0).float().mean()) > 0.3 and float(img[:, 12:].abs().max()) < 0.45
    pcd = torch.from_numpy(gbuffer.read_fps_pcd(PLY)[:512])[None]
    sd = ve.random_state_dict(seed=0)
    start = torch.tensor([17])
    noise = torch.randn(1, K, 10, generator=torch.Generator().manual_seed(2))
    enc = ve.SurfelEncoder(sd, num_frames=V, latent_num=K)
    enc.use_graph = False
    out = enc.encode(img, pcd.to(DEV), start, noise=noise.to(DEV))
    torch.cuda.synchronize()
    want = vo.encode(sd, img.cpu(), pcd, V, K, start, emulate_bf16=True)
    post = vo.posterior(sd, want["h"], noise)
    rel = lambda a, b: float((a.double().cpu() - b.double()).norm() / b.double().norm())
    assert torch.equal(out["fps_idx"].cpu().long(), want["fps_idx"])
    errs = {"h": rel(out["h"], want["h"]), "mean": rel(out["mean"], post["mean"]),
            "logvar": rel(out["logvar"], post["logvar"])}
    print("encoder on a real chunk input vs bf16 oracle rel-L2:", errs)
    for k, e in errs.items():
        assert e <= 6e-3, (k, e)


def test_reconstruct_chunk_end_to_end(chunk):
    from gaussiananything_b200 import gbuffer
    from gaussiananything_b200 import vae_decoder as vd
    from gaussiananything_b200 import vae_encoder as ve
    dec = vd.SurfelDecoder(vd.random_state_dict(D=768, depth=2), num_heads=12, depth=2)
    enc = ve.SurfelEncoder(ve.random_state_dict(seed=3), num_frames=8, latent_num=768)
    ae = vd.SurfelAE(dec, encoder=enc)
    out = ae(behaviour="reconstruct_chunk", chunk=CHUNK, pcd=PLY, fps_start=torch.tensor([5]),
             generator=torch.Generator().manual_seed(0))
    torch.cuda.synchronize()
    assert out["gaussians_upsampled_3"].shape == (1, 96 * 768, 13) and out["latent_normalized"].shape == (1, 768, 10)
    assert out["input"]["views"] == list(range(8)) and out["eval"]["views"] == list(range(8, 16))
    for part, views in (("input", range(8)), ("eval", range(8, 16))):
        p = out[part]
        assert p["render"]["image"].shape == (1, 8, 3, 512, 512) and p["table"].shape == (8, 8)
        assert torch.equal(p["c"].cpu(), torch.from_numpy(chunk["c"][list(views)]))
        assert all(torch.isfinite(v).all() for v in p["metrics"].values())
        want = go.metric_table({k: v[0] for k, v in p["render"].items()}, p["targets"])
        got = p["table"].double().cpu()
        assert float(((got - want).abs() / want.abs().clamp_min(1.0)).max()) <= 1e-5
        assert torch.equal(p["targets"]["depth"].cpu()[:, 0], torch.from_numpy(chunk["depth"][list(views)]))
    # a second call from the decoded chunk and points, with the same seeds: the same Gaussians
    again = ae(behaviour="reconstruct_chunk", chunk=chunk, pcd=gbuffer.read_fps_pcd(PLY), fps_start=torch.tensor([5]),
               generator=torch.Generator().manual_seed(0))
    assert torch.equal(again["gaussians_upsampled_3"], out["gaussians_upsampled_3"])
    with pytest.raises(ValueError, match="8"):
        ae(behaviour="reconstruct_chunk", chunk=chunk, pcd=PLY, input_views=range(4))
    with pytest.raises(NotImplementedError):
        vd.SurfelAE(dec)(behaviour="reconstruct_chunk", chunk=chunk, pcd=PLY)
