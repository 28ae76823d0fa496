"""GPU mesh export against oracle/tsdf_oracle.py stage by stage, the sphere known answer on the GPU mesh, determinism,
input validation and the end-to-end export."""
import numpy as np
import pytest
import torch

from gaussiananything_b200 import mesh
from oracle import tsdf_oracle as to
from tests import mesh_scenes as ms

pytestmark = pytest.mark.gpu


def _compare(rgb, depth, alpha, setup, alpha_thres=0.08):
    """Runs both fusions on the same maps (device maps copied to the host for the oracle) and checks every stage."""
    m, st = mesh.fuse(rgb, depth, alpha, setup, alpha_thres=alpha_thres)
    torch.cuda.synchronize()
    o = to.fuse(rgb.cpu().numpy(), depth.cpu().numpy(), alpha.cpu().numpy(), setup, alpha_thres=alpha_thres)
    assert np.array_equal(st["texels"].cpu().numpy(), to.texels(o["depth"], o["rgb8"]))
    V = rgb.shape[0]
    tab = st["table"].cpu().numpy().view(np.uint32)
    bits = np.stack([(tab[:, v >> 5] >> (v & 31)) & 1 for v in range(V)]).astype(bool)
    assert np.array_equal(bits, o["touched"])
    assert np.array_equal(st["pool"].cpu().numpy(), o["pool"])
    vox = st["voxels"].cpu().numpy()
    assert np.array_equal(vox[1], o["state"][1])                       # weights
    assert np.array_equal(vox[0], o["state"][0]) and np.array_equal(vox[2:], o["state"][2:])
    assert np.array_equal(st["cube"][0].cpu().numpy(), o["cube"])
    assert m.vertices.shape == o["vertices"].shape and m.triangles.shape == o["triangles"].shape
    assert np.abs(m.vertices - o["vertices"]).max(initial=0) <= 1e-9
    assert np.abs(m.vertex_colors - o["colors"]).max(initial=0) <= 1e-9
    assert np.array_equal(m.triangles, o["triangles"])
    label, sizes = mesh.clusters(m)
    ol, osz = to.clusters(o["triangles"])
    assert np.array_equal(sizes.cpu().numpy(), osz) and np.array_equal(label.cpu().numpy(), ol)
    post = mesh.post_process_mesh(m)
    pv, pc, pt, *_ = to.post_process(o["vertices"], o["colors"], o["triangles"])
    assert np.array_equal(post.triangles, pt)
    assert np.abs(post.vertices - pv).max(initial=0) <= 1e-9
    return m, o


def _sphere(size, views):
    p = mesh.uni_mesh_path(10)[views]
    rgb, d, a = ms.sphere_maps(p, size)
    dev = torch.device("cuda")
    return p, torch.tensor(rgb, device=dev), torch.tensor(d, device=dev), torch.tensor(a, device=dev)


def test_stages_match_oracle_analytic_128():
    p, rgb, d, a = _sphere(128, slice(0, 50, 4))                      # 13 views
    _compare(rgb, d, a, mesh.view_setup(p, 128, 128))


@pytest.mark.parametrize("alpha_thres", [0.08, 0.6])
def test_stages_match_oracle_rasterised_128(alpha_thres):
    p = mesh.uni_mesh_path(10)[::4][:12]
    g = torch.tensor(ms.surface_surfels(20000, 1), device="cuda")
    _, out = mesh.render_orbit(g, p, 128)
    _compare(out["image"][0], out["depth"][0, :, 0], out["alpha"][0, :, 0], mesh.view_setup(p, 128, 128),
             alpha_thres)


@pytest.mark.parametrize("name", sorted(ms.post_process_cases()))
def test_post_process_hand_built_meshes_match_oracle(name):
    """Ties at the threshold, bow-ties, degenerate triangles and unreferenced vertices through the GPU filter."""
    v, c, t = ms.post_process_cases()[name]
    got = mesh.post_process_mesh(mesh.TriangleMesh(v, t.astype(np.int32), c))
    pv, pc, pt, label, sizes, _ = to.post_process(v, c, t)
    assert np.array_equal(got.triangles, pt)
    assert np.array_equal(got.vertices, pv) and np.array_equal(got.vertex_colors, pc)
    gl, gs = mesh.clusters(mesh.TriangleMesh(v, t.astype(np.int32), c))
    assert np.array_equal(gs.cpu().numpy(), sizes) and np.array_equal(gl.cpu().numpy(), label)


def test_post_process_rejects_bad_meshes():
    v, c, t = ms.post_process_cases()["ties"]
    for bad in (t.max() + 1, -1):
        t2 = t.astype(np.int32).copy()
        t2[5, 1] = bad
        with pytest.raises(ValueError, match="triangle index"):
            mesh.post_process_mesh(mesh.TriangleMesh(v, t2, c))
        with pytest.raises(ValueError, match="triangle index"):
            mesh.clusters(mesh.TriangleMesh(v, t2, c))
    with pytest.raises(ValueError):
        mesh.post_process_mesh(mesh.TriangleMesh(v, t.astype(np.int32), c[:-1]))


def test_deployed_size_matches_oracle():
    g = torch.tensor(ms.surface_surfels(73728, 0), device="cuda")
    p, out = mesh.render_orbit(g, None, 512)
    m, o = _compare(out["image"][0], out["depth"][0, :, 0], out["alpha"][0, :, 0], mesh.view_setup(p, 512, 512))
    assert len(m.triangles) > 10000


def test_sphere_known_answer_on_gpu():
    p, rgb, d, a = _sphere(512, slice(None))
    m = mesh.extract_mesh_bounded([rgb[i:i + 1] for i in range(50)], [d[i:i + 1, None] for i in range(50)],
                                  [a[i:i + 1, None] for i in range(50)], p)
    ms.check_sphere_mesh(m.vertices, m.triangles, m.vertex_colors, mesh.volume_settings()[2], within_half=0.98)


def test_deterministic_bytes():
    p, rgb, d, a = _sphere(128, slice(0, 50, 3))
    s = mesh.view_setup(p, 128, 128)
    m1, m2 = mesh.fuse(rgb, d, a, s)[0], mesh.fuse(rgb, d, a, s)[0]
    p1, p2 = mesh.post_process_mesh(m1), mesh.post_process_mesh(m2)
    for x, y in ((m1, m2), (p1, p2)):
        assert x.vertices.tobytes() == y.vertices.tobytes() and x.triangles.tobytes() == y.triangles.tobytes()
        assert x.vertex_colors.tobytes() == y.vertex_colors.tobytes()


def test_input_validation_and_out_of_box():
    p, rgb, d, a = _sphere(64, slice(0, 4))
    s = mesh.view_setup(p, 64, 64)
    with pytest.raises(ValueError):
        mesh.fuse(rgb, d[:, :32], a, s)
    with pytest.raises(RuntimeError, match="CUDA"):
        mesh.fuse(rgb, d.cpu(), a, s)
    with pytest.raises(TypeError):
        mesh.fuse(rgb, d, a.double(), s)
    with pytest.raises(TypeError):
        mesh.extract_mesh_bounded([x[None] for x in rgb.double()], [x[None, None] for x in d],
                                  [x[None, None] for x in a], p)
    with pytest.raises(RuntimeError):
        mesh.extract_mesh_bounded([x[None] for x in rgb.cpu()], [x[None, None] for x in d.cpu()],
                                  [x[None, None] for x in a.cpu()], p)
    small = dict(s, box=np.array([-2, -2, -2, 4, 4, 4], np.int32))    # the sphere's far side leaves this box
    guard = torch.full((1 << 20,), 7, dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError, match="outside the volume box"):
        mesh.fuse(rgb, d, a, small)
    assert int((guard != 7).sum()) == 0
    m, _ = mesh.fuse(rgb, d, a, s)                                   # still fine afterwards
    assert len(m.triangles) > 0


def test_end_to_end_export(tmp_path):
    g = torch.tensor(ms.surface_surfels(73728, 0), device="cuda")
    rgbs, depths, alphas, cams, m = mesh.mesh_from_surfels(g)
    path = mesh.export_mesh_from_2dgs(rgbs, depths, alphas, cams, 0, 0, output_dir=str(tmp_path))
    assert path == str(tmp_path / "0" / "0-mesh.obj")
    raw = mesh.read_triangle_mesh(str(tmp_path / "0" / "0-mesh_raw.obj"))
    post = mesh.read_triangle_mesh(path)
    assert np.abs(raw.vertices - m.vertices).max() <= 1e-12 and np.array_equal(raw.triangles, m.triangles)
    assert 0 < len(post.triangles) <= len(raw.triangles)
