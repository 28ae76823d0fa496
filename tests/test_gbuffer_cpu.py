"""G-buffer chunk front end without a GPU: the chunk and PLY readers, the oracle against the golden the reference's own
read_chunk and PostProcess._post_process_sample_batch produced (tests/golden/make_gbuffer_golden.py), the metric
definitions, the argument checks, and the compiler's report on csrc/gbuffer_ops.cu."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import gbuffer_oracle as go

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
CHUNK = os.path.join(GOLDEN, "gbuffer_chunk")


@pytest.fixture(scope="module")
def chunk():
    from gaussiananything_b200 import gbuffer
    return gbuffer.read_chunk(CHUNK)


@pytest.fixture(scope="module")
def gold():
    with np.load(os.path.join(GOLDEN, "gbuffer_small.npz")) as z:
        return {k: z[k] for k in z.files}


def test_read_chunk_shapes_and_dtypes(chunk):
    want = {"raw_img": ((512, 8192, 3), np.uint8), "normal": ((512, 8192, 3), np.uint8), "alpha": ((512, 8192), np.uint8),
            "depth": ((16, 512, 512), np.float32), "c": ((16, 25), np.float32), "bbox": ((16, 4), np.uint8)}
    for k, (shape, dtype) in want.items():
        assert chunk[k].shape == shape and chunk[k].dtype == dtype, k
    assert chunk["ins"] == "Animals/0/10075" and chunk["caption"].startswith("a green lizard")
    assert float(chunk["depth"].min()) == 0.0 and 0.05 < float((chunk["depth"] > 0).mean()) < 0.6


def test_read_chunk_names_what_is_wrong(tmp_path, chunk):
    from gaussiananything_b200 import gbuffer
    for f in ("raw_img.jpg", "c.npy", "alpha.jpg", "normal.png"):
        shutil.copy(os.path.join(CHUNK, f), tmp_path / f)
    with pytest.raises(FileNotFoundError, match="depth.npz"):
        gbuffer.read_chunk(str(tmp_path))
    np.savez(tmp_path / "depth.npz", depth=np.zeros((16, 256, 256), np.float32))
    with pytest.raises(ValueError, match=r"raw_img.jpg is \(512, 8192, 3\)"):
        gbuffer.read_chunk(str(tmp_path))
    small = dict(chunk, depth=chunk["depth"][:, :256, :256])
    with pytest.raises(NotImplementedError, match="256 x 256"):
        gbuffer.pack(small, range(8))
    with pytest.raises(IndexError, match="16"):
        gbuffer.pack(chunk, [3, 16])
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        gbuffer.pack(chunk, range(8), device="cpu")


def test_read_fps_pcd_both_encodings(tmp_path):
    from gaussiananything_b200 import gbuffer
    pts = gbuffer.read_fps_pcd(os.path.join(CHUNK, "fps-4096.ply"))                 # binary_little_endian
    assert pts.shape == (4096, 3) and pts.dtype == np.float32
    assert float(np.abs(pts).max()) <= 0.45 + 1e-6 and float(pts.std()) > 0.02
    head = "ply\nformat ascii 1.0\ncomment made by hand\nelement vertex 5\nproperty float x\nproperty float y\n" \
           "property float z\nproperty uchar red\nelement face 0\nproperty list uchar int vertex_indices\nend_header\n"
    rows = "".join("%r %r %r %d\n" % (float(x), float(y), float(z), i) for i, (x, y, z) in enumerate(pts[:5]))
    (tmp_path / "a.ply").write_text(head + rows)
    assert np.array_equal(gbuffer.read_fps_pcd(str(tmp_path / "a.ply")), pts[:5])
    # extra vertex properties and a double-typed coordinate in the binary form
    dt = np.dtype([("x", "<f8"), ("y", "<f4"), ("nx", "<f4"), ("z", "<f4")])
    v = np.zeros(5, dt)
    v["x"], v["y"], v["z"] = pts[:5, 0], pts[:5, 1], pts[:5, 2]
    head = b"ply\nformat binary_little_endian 1.0\nelement vertex 5\nproperty double x\nproperty float y\n" \
           b"property float nx\nproperty float z\nend_header\n"
    (tmp_path / "b.ply").write_bytes(head + v.tobytes())
    assert np.array_equal(gbuffer.read_fps_pcd(str(tmp_path / "b.ply")), pts[:5])
    (tmp_path / "c.ply").write_bytes(head + v.tobytes()[:-8])
    with pytest.raises(ValueError, match="holds fewer"):
        gbuffer.read_fps_pcd(str(tmp_path / "c.ply"))
    (tmp_path / "d.ply").write_bytes(head.replace(b"little", b"big") + v.tobytes())
    with pytest.raises(ValueError, match="binary_big_endian"):
        gbuffer.read_fps_pcd(str(tmp_path / "d.ply"))
    (tmp_path / "e.ply").write_bytes(b"solid not a ply\n")
    with pytest.raises(ValueError, match="not a PLY"):
        gbuffer.read_fps_pcd(str(tmp_path / "e.ply"))


def _sub(t, gold):
    s, o = int(gold["stride"]), int(gold["offset"])
    return t[..., o::s, o::s]


def test_oracle_fp32_reproduces_the_reference(chunk, gold):
    """float32 mode repeats the reference's operations: channels 0-5 and the targets bit for bit, rays and xyz within
    1e-6, and the set of zeroed xyz values identical at every pixel of all 16 views."""
    got = go.pack(chunk, dtype=torch.float32)
    enc = got["img_to_encoder"]
    assert enc.dtype == torch.float32 and tuple(enc.shape) == (16, 15, 512, 512)
    e, g = _sub(enc, gold).numpy(), gold["img_to_encoder"]
    assert np.array_equal(e[:, :6], g[:, :6])
    assert float(np.abs(e[:, 6:] - g[:, 6:]).max()) <= 1e-6
    for k in ("img", "alpha", "depth"):
        assert np.array_equal(_sub(got[k], gold).numpy().reshape(gold[k].shape), gold[k]), k
    assert np.array_equal(got["c"].numpy(), gold["c"])
    zero = np.unpackbits(gold["xyz_zero_bits"]).reshape(16, 3, 512, 512).astype(bool)
    assert np.array_equal(enc[:, 12:15].numpy() == 0, zero)
    # the structure a real input has: background is zeroed only where the camera origin is outside the clip
    assert 0.3 < zero.mean() < 0.95 and float(np.abs(e[:, 12:]).max()) < 0.45


def test_oracle_fp64_is_within_rounding_of_the_reference(chunk, gold):
    """float64 mode (the kernel's yardstick) against the fp32 reference: 1e-6 absolute on rays and xyz, except where
    an fp64 coordinate is within 1e-6 of the clip value and the zero rule may fall either way."""
    got = go.pack(chunk, dtype=torch.float64)
    e, g = _sub(got["img_to_encoder"], gold).numpy(), gold["img_to_encoder"].astype(np.float64)
    assert np.array_equal(e[:, :6], g[:, :6])
    assert float(np.abs(e[:, 6:12] - g[:, 6:12]).max()) <= 1e-6
    d = np.abs(e[:, 12:] - g[:, 12:])
    odd = d > 1e-6
    assert odd.mean() < 1e-4
    assert np.all((e[:, 12:][odd] == 0) | (g[:, 12:][odd] == 0)), "only the zero rule may differ"
    assert float(np.abs(np.where(e[:, 12:][odd] == 0, g[:, 12:][odd], e[:, 12:][odd])).min(initial=1.0)) > 0.45 - 2e-6


def test_subset_of_views_and_view_order(chunk):
    views = [9, 2, 15]
    a, full = go.pack(chunk, views, torch.float32), go.pack(chunk, None, torch.float32)
    for k in ("img_to_encoder", "img", "alpha", "depth", "mask", "c"):
        assert torch.equal(a[k], full[k][views]), k


def test_two_ray_conventions_differ_only_in_rounding(chunk):
    """gen_rays (Pluecker) and RaySampler (unprojection) describe the same ray; they are computed differently and the
    kernel keeps both, so this pins the claim the header makes."""
    c = chunk["c"][[1, 6]]
    d1 = torch.stack([go.pluecker(ci, 64)[3:] for ci in c]).permute(0, 2, 3, 1).reshape(2, -1, 3)
    o, d2 = go.sampler_rays(c, 64)
    assert float((d1 - d2).abs().max()) < 1e-6                   # c.npy is fp32, so c2w is orthonormal to ~1e-7
    m = torch.stack([go.pluecker(ci, 64)[:3] for ci in c]).permute(0, 2, 3, 1).reshape(2, -1, 3)
    assert float((m - torch.cross(o[:, None].expand_as(d2), d2, dim=-1)).abs().max()) < 1e-6


def _fake_render(t, g, noise):
    """A render dict [V, ...] near the targets."""
    V = t["img"].shape[0]
    r = lambda *s: torch.rand(*s, generator=g)
    return {"image": ((t["img"] + 1) / 2 + noise * (r(V, 3, 64, 64) - 0.5)).clamp(0, 1),
            "depth": t["depth"] + noise * r(V, 1, 64, 64), "alpha": (t["alpha"] + noise * (r(V, 1, 64, 64) - 0.5)).clamp(0, 1),
            "rend_normal": torch.nn.functional.normalize(t["normal"] + noise * (r(V, 3, 64, 64) - 0.5), dim=1)}


def test_metric_definitions(chunk):
    full = go.pack(chunk, [0, 5, 9], torch.float32)
    t = {k: full[k][..., 100:356:4, 100:356:4].contiguous() for k in ("img", "alpha", "depth", "mask")}
    t["normal"] = full["img_to_encoder"][:, 3:6, 100:356:4, 100:356:4].contiguous()
    for k in ("alpha", "depth", "mask"):                                            # view 2: all background
        t[k][2] = 0
    g = torch.Generator().manual_seed(0)
    m = go.derive(go.metric_table(_fake_render(t, g, 0.1), t))
    assert all(torch.isfinite(v).all() for v in m.values())
    assert 20 < float(m["psnr"][0]) < 40 and 0.04 < float(m["depth_l1"][0]) < 0.06
    assert float(m["fg_pixels"][2]) == 0 and float(m["depth_l1"][2]) == 0 and float(m["normal_error"][2]) == 0
    # the targets as the prediction: no error, except that 8-bit normals are not unit length (1 - |n|^2 remains)
    same = {"image": (t["img"] + 1) / 2, "depth": t["depth"], "alpha": t["alpha"], "rend_normal": t["normal"]}
    m = go.derive(go.metric_table(same, t))
    assert torch.all(m["psnr"] == go.PSNR_CAP) and torch.all(m["depth_l1"] == 0) and torch.all(m["alpha_l1"] == 0)
    assert torch.all(m["iou"] == 1) and float(m["normal_error"].abs().max()) < 0.02
    empty = dict(same, alpha=torch.zeros_like(t["alpha"]))
    assert float(go.derive(go.metric_table(empty, dict(t, alpha=torch.zeros_like(t["alpha"]))))["iou"][0]) == 1.0
    from gaussiananything_b200 import gbuffer
    tab = go.metric_table(_fake_render(t, g, 0.1), t)
    a, b = gbuffer.derive(tab), go.derive(tab)
    assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
    assert gbuffer.METRIC_BLOCKS == int(re.search(r"#define GA_RECON_METRICS_BLOCKS\s+(\d+)",
                                                  open(os.path.join(ROOT, "include", "ga_b200.h")).read()).group(1))


def test_cameras_share_the_orbit_conversion(chunk):
    from gaussiananything_b200 import gbuffer, mesh
    cam = gbuffer.cameras(chunk["c"][8:])
    view, proj, pos, tanfov = mesh.orbit_cameras(chunk["c"][8:])
    assert torch.equal(cam["cam_view"], view) and torch.equal(cam["cam_view_proj"], proj)
    assert torch.equal(cam["cam_pos"], pos) and cam["tanfov"] == tanfov and tuple(view.shape) == (1, 8, 4, 4)
    assert float((pos[0] - torch.from_numpy(chunk["c"][8:, [3, 7, 11]])).abs().max()) < 1e-6
    assert abs(tanfov - 0.5 / float(chunk["c"][8, 16])) < 1e-6


def test_reconstruct_chunk_needs_an_encoder():
    from gaussiananything_b200.vae_decoder import SurfelAE
    ae = SurfelAE.__new__(SurfelAE)
    ae.encoder = None
    with pytest.raises(NotImplementedError, match="encoder="):
        ae.forward(behaviour="reconstruct_chunk", chunk=CHUNK, pcd=os.path.join(CHUNK, "fps-4096.ply"))


def test_kernels_compile_without_spills(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    from gaussiananything_b200 import build
    src = os.path.join(build.CSRC, "gbuffer_ops.cu")
    assert build.EXTRA["gbuffer_ops.cu"] == ["--fmad=false"]
    r = subprocess.run([nvcc] + build.ARCH + build.COMMON + build.EXTRA["gbuffer_ops.cu"] +
                       ["-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "g.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    regs = [int(x) for x in re.findall(r"Used (\d+) registers", r.stderr)]
    assert len(spills) == 3 and all(s == ("0", "0") for s in spills), r.stderr
    assert max(regs) <= 128, regs                    # 256-thread blocks: two or more resident per SM
