"""GPU parity tests of the surfel rasteriser: CUDA path (through the C ABI)
against the CPU oracle on identical seeded inputs.

Bars (SURVEY.md 8d / BASELINE.json north_star): integer tile/bin indices
bit-exact; rendered RGB-D(+alpha, normal, distortion) rel-L2 <= 1e-3;
gradients rel-L2 <= 1e-3.  The oracle itself is PARITY UNPINNED (upstream
rasteriser not vendored, no reference tests) -- see oracle/surfel_oracle.c.
"""
import numpy as np
import pytest
import torch

from tests.helpers import cameras, oracle_view, rel_l2, scene

pytestmark = pytest.mark.gpu

TOL = 1e-3


def _run_cuda(g, views, projs, bg, H, W, scale_modifier=1.0, batch=1):
    from gaussiananything_b200 import raster
    dev = torch.device("cuda:0")
    P = g.shape[-2]
    g13 = torch.tensor(g, device=dev).reshape(batch, P, 13)
    V = views.shape[0] // batch
    vm = torch.tensor(views, device=dev).reshape(batch, V, 4, 4)
    pm = torch.tensor(projs, device=dev).reshape(batch, V, 4, 4)
    bgt = torch.tensor(bg, dtype=torch.float32, device=dev)
    color, allmap, radii, state = raster.forward_raw(g13, vm, pm, bgt, H, W, scale_modifier)
    wsv = raster.workspace_views(state["ws"], state["L"], batch, P, V, H, W, state["max_instances"])
    return color, allmap, radii, state, wsv


def _check_view(o, color, allmap, radii, wsv, nv, P, H, W, tol=TOL):
    T = ((W + 15) // 16) * ((H + 15) // 16)
    # --- integers: bit exact
    assert np.array_equal(radii.cpu().numpy(), o["radii"]), "radii differ"
    rect = wsv["rect"][nv].cpu().numpy().astype(np.uint32)
    orect = o["rect"].astype(np.uint32)
    packed = orect[:, 0] | (orect[:, 1] << 8) | (orect[:, 2] << 16) | (orect[:, 3] << 24)
    assert np.array_equal(rect, packed), "tile rects differ"
    assert np.array_equal(wsv["depth"][nv].cpu().numpy().view(np.uint32), o["depth"].view(np.uint32)), "depth bits differ"
    ts = wsv["tile_start"].cpu().numpy()[nv * T:(nv + 1) * T + 1].astype(np.int64)
    base = ts[0]
    rng = o["ranges"].astype(np.int64)
    cnt = rng[:, 1] - rng[:, 0]
    assert np.array_equal(ts[1:] - ts[:-1], cnt), "tile ranges differ"
    D = o["num_rendered"]
    ids = wsv["ids"].cpu().numpy()[base:base + D].astype(np.uint32)
    assert np.array_equal(ids, o["ids"]), "sorted surfel ids differ"
    keys = wsv["keys"].cpu().numpy()[base:base + D].view(np.uint64)
    assert np.array_equal((keys >> np.uint64(32)).astype(np.uint32), (o["keys"] & np.uint64(0xffffffff)).astype(np.uint32)), "depth keys differ"
    # --- floats
    c = color.cpu().numpy(); a = allmap.cpu().numpy()
    assert rel_l2(c, o["color"]) <= tol, ("color", rel_l2(c, o["color"]))
    for ch, name in enumerate(["depth", "alpha", "nx", "ny", "nz", "median_depth", "distortion"]):
        if np.linalg.norm(o["allmap"][ch]) == 0:
            assert np.abs(a[ch]).max() <= 1e-6
            continue
        r = rel_l2(a[ch], o["allmap"][ch])
        if name == "median_depth":
            # a pixel whose T crosses 0.5 within rounding picks a different surfel: bound the count
            bad = np.abs(a[ch] - o["allmap"][ch]) > 1e-4 * np.maximum(1.0, np.abs(o["allmap"][ch]))
            assert bad.mean() <= 2e-4, (name, bad.mean())
        elif name == "distortion":
            # sum_ij w_i w_j (m_i-m_j)^2 is evaluated as m^2 A + M2 - 2 m M1: it cancels when depths
            # coincide, so accept a small absolute error too (m in [0,1], weights sum <= 1)
            assert r <= tol or np.abs(a[ch] - o["allmap"][ch]).max() <= 2e-5, (name, r)
        else:
            assert r <= tol, (name, r)
    nc = wsv["n_contrib"][nv].cpu().numpy()
    mism = (nc[0] != o["n_contrib"][0]).mean()
    assert mism <= 2e-4, ("n_contrib mismatch rate", mism)


@pytest.mark.parametrize("P,H,W,boost,seed", [
    (10000, 256, 256, 1.0, 0),      # BASELINE config C1 shape
    (3000, 250, 300, 8.0, 1),       # ragged image, larger splats
    (500, 64, 48, 40.0, 2),         # big splats: many tiles each, early termination
    (1, 32, 32, 40.0, 3),           # single surfel
    (4000, 128, 128, 1.0, 4),
])
def test_forward_parity_single_view(P, H, W, boost, seed):
    g = scene(P, seed, boost)
    vs, ps, _, _ = cameras(1, start=seed)
    bg = [1.0, 0.5, 0.2]
    color, allmap, radii, state, wsv = _run_cuda(g, vs, ps, bg, H, W)
    o = oracle_view(g, vs[0], ps[0], bg, H, W)
    assert state["num_rendered"] == o["num_rendered"]
    _check_view(o, color[0, 0], allmap[0, 0], radii[0, 0], wsv, 0, P, H, W)


def test_forward_parity_batched_views_and_batches():
    B, V, P, H, W = 2, 3, 2500, 160, 144
    g = np.stack([scene(P, 10, 6.0), scene(P, 11, 3.0)])
    vs, ps, _, _ = cameras(B * V)
    bg = [1.0, 1.0, 1.0]
    color, allmap, radii, state, wsv = _run_cuda(g, vs, ps, bg, H, W, batch=B)
    tot = 0
    for b in range(B):
        for v in range(V):
            nv = b * V + v
            o = oracle_view(g[b], vs[nv], ps[nv], bg, H, W)
            tot += o["num_rendered"]
            _check_view(o, color[b, v], allmap[b, v], radii[b, v], wsv, nv, P, H, W)
    assert tot == state["num_rendered"]


def test_all_culled_and_empty_tiles():
    P, H, W = 256, 64, 64
    g = scene(P, 5)
    g[:, 0:3] += 100.0          # far outside the frustum / behind the camera for some views
    vs, ps, _, _ = cameras(1)
    bg = [0.25, 0.5, 0.75]
    color, allmap, radii, state, wsv = _run_cuda(g, vs, ps, bg, H, W)
    o = oracle_view(g, vs[0], ps[0], bg, H, W)
    assert state["num_rendered"] == o["num_rendered"]
    assert np.array_equal(radii[0, 0].cpu().numpy(), o["radii"])
    assert rel_l2(color[0, 0].cpu().numpy(), o["color"]) <= 1e-6


def test_scale_modifier_and_low_opacity():
    P, H, W = 2000, 96, 96
    g = scene(P, 6, 10.0)
    g[::3, 3] = 0.001           # below 1/255: stays in the lists, never contributes
    vs, ps, _, _ = cameras(1)
    bg = [0.0, 0.0, 0.0]
    color, allmap, radii, state, wsv = _run_cuda(g, vs, ps, bg, H, W, scale_modifier=1.7)
    o = oracle_view(g, vs[0], ps[0], bg, H, W, scale_modifier=1.7)
    _check_view(o, color[0, 0], allmap[0, 0], radii[0, 0], wsv, 0, P, H, W)


def test_sort_fallback_large_tile():
    # > 4096 instances in one tile -> the global-memory sort path
    P, H, W = 6000, 32, 32
    g = scene(P, 7, 1.0)
    g[:, 0:3] *= 0.02
    vs, ps, _, _ = cameras(1)
    bg = [1.0, 1.0, 1.0]
    color, allmap, radii, state, wsv = _run_cuda(g, vs, ps, bg, H, W)
    o = oracle_view(g, vs[0], ps[0], bg, H, W)
    assert int(wsv["status"][2]) >= 1, "expected at least one tile on the fallback sort"
    _check_view(o, color[0, 0], allmap[0, 0], radii[0, 0], wsv, 0, P, H, W)


def test_workspace_overflow_retry():
    from gaussiananything_b200 import raster
    P, H, W = 3000, 128, 128
    g = scene(P, 8, 20.0)
    vs, ps, _, _ = cameras(1)
    dev = torch.device("cuda:0")
    g13 = torch.tensor(g, device=dev)[None]
    vm = torch.tensor(vs, device=dev)[None]
    pm = torch.tensor(ps, device=dev)[None]
    bg = torch.ones(3, device=dev)
    c1, a1, r1, s1 = raster.forward_raw(g13, vm, pm, bg, H, W, max_instances=16)   # forces a retry
    o = oracle_view(g, vs[0], ps[0], [1, 1, 1], H, W)
    assert s1["num_rendered"] == o["num_rendered"]
    assert rel_l2(c1[0, 0].cpu().numpy(), o["color"]) <= TOL


@pytest.mark.parametrize("P,H,W,boost,seed,V", [
    (2000, 96, 112, 10.0, 20, 1),
    (800, 64, 64, 40.0, 21, 2),
    (10000, 256, 256, 1.0, 22, 1),
])
def test_backward_parity(P, H, W, boost, seed, V):
    from gaussiananything_b200 import raster
    from oracle import surfel_oracle as so
    g = scene(P, seed, boost)
    vs, ps, _, _ = cameras(V, start=seed)
    bg = [1.0, 0.5, 0.2]
    dev = torch.device("cuda:0")
    g13 = torch.tensor(g, device=dev)[None].requires_grad_(True)
    vm = torch.tensor(vs, device=dev)[None]
    pm = torch.tensor(ps, device=dev)[None]
    color, allmap, radii = raster.rasterize_surfels_batched(g13, vm, pm, torch.tensor(bg, device=dev), H, W, 1.0)
    rng = np.random.default_rng(seed)
    gc = rng.standard_normal((V, 3, H, W)).astype(np.float32)
    ga = rng.standard_normal((V, 7, H, W)).astype(np.float32)
    loss = (color[0] * torch.tensor(gc, device=dev)).sum() + (allmap[0] * torch.tensor(ga, device=dev)).sum()
    loss.backward()
    got = g13.grad[0].cpu().numpy().astype(np.float64)
    want = np.zeros((P, 13))
    for v in range(V):
        o = oracle_view(g, vs[v], ps[v], bg, H, W)
        b = so.rasterize_backward(o, gc[v], ga[v])
        want[:, 0:3] += b["means3D"]; want[:, 3:4] += b["opacities"]; want[:, 4:6] += b["scales"]
        want[:, 6:10] += b["rotations"]; want[:, 10:13] += b["colors"]
    for name, sl in [("means3D", slice(0, 3)), ("opacity", slice(3, 4)), ("scales", slice(4, 6)),
                     ("rotations", slice(6, 10)), ("colors", slice(10, 13))]:
        r = rel_l2(got[:, sl], want[:, sl])
        assert r <= TOL, (name, r)


def test_reference_api_surface():
    """diff_surfel_rasterization / GaussianRenderer2DGS mirrors give the same pixels as the batched call."""
    from gaussiananything_b200.diff_surfel_rasterization import GaussianRasterizationSettings, GaussianRasterizer
    from gaussiananything_b200.gs_surfel import GaussianRenderer2DGS
    P, H = 3000, 128
    g = scene(P, 30, 5.0)
    vs, ps, cs, tf = cameras(2)
    dev = torch.device("cuda:0")
    gt = torch.tensor(g, device=dev)
    bg = torch.tensor([1.0, 1.0, 1.0], device=dev)
    rs = GaussianRasterizationSettings(image_height=H, image_width=H, tanfovx=tf, tanfovy=tf, bg=bg,
                                       scale_modifier=1.0, viewmatrix=torch.tensor(vs[0], device=dev),
                                       projmatrix=torch.tensor(ps[0], device=dev), sh_degree=0,
                                       campos=torch.tensor(cs[0], device=dev), prefiltered=False, debug=False)
    rast = GaussianRasterizer(raster_settings=rs)
    img, radii, allmap = rast(means3D=gt[:, 0:3], means2D=torch.zeros_like(gt[:, 0:3]), shs=None,
                              colors_precomp=gt[:, 10:13], opacities=gt[:, 3:4], scales=gt[:, 4:6],
                              rotations=gt[:, 6:10], cov3D_precomp=None)
    assert img.shape == (3, H, H) and allmap.shape == (7, H, H) and radii.shape == (P,)
    assert radii.dtype == torch.int32
    o = oracle_view(g, vs[0], ps[0], [1, 1, 1], H, H)
    assert rel_l2(img.cpu().numpy(), o["color"]) <= TOL
    with pytest.raises(Exception):
        rast(means3D=gt[:, 0:3], means2D=None, opacities=gt[:, 3:4], shs=None, colors_precomp=None,
             scales=gt[:, 4:6], rotations=gt[:, 6:10])
    r = GaussianRenderer2DGS(H, 3, {})
    out = r.render(gt[None], torch.tensor(vs, device=dev)[None], torch.tensor(ps, device=dev)[None],
                   torch.tensor(cs, device=dev)[None], tf)
    assert out["image"].shape == (1, 2, 3, H, H) and out["rend_normal"].shape == (1, 2, 3, H, H)
    assert out["alpha"].shape == (1, 2, 1, H, H) and out["depth"].shape == (1, 2, 1, H, H)
    assert rel_l2(out["image"][0, 0].cpu().numpy(), np.clip(o["color"], 0, 1)) <= TOL
    # normals rotated camera->world exactly like the reference post-processing (gs_surfel.py:125-128)
    n_ref = np.einsum('chw,dc->dhw', o["allmap"][2:5], vs[0][:3, :3])
    assert rel_l2(out["rend_normal"][0, 0].cpu().numpy(), n_ref) <= TOL


def test_full_size_properties():
    """BASELINE config C2 size (100k surfels, 512^2, 6 views): size-independent properties."""
    from gaussiananything_b200 import raster
    P, H, W, V = 100000, 512, 512, 6
    g = scene(P, 40)
    vs, ps, _, _ = cameras(V)
    dev = torch.device("cuda:0")
    g13 = torch.tensor(g, device=dev)[None]
    vm = torch.tensor(vs, device=dev)[None]
    pm = torch.tensor(ps, device=dev)[None]
    bg = torch.ones(3, device=dev)
    c1, a1, r1, s1 = raster.forward_raw(g13, vm, pm, bg, H, W)
    # 1. batched == per-view calls, bit for bit (views are independent)
    for v in (0, 5):
        c2, a2, r2, s2 = raster.forward_raw(g13, vm[:, v:v + 1], pm[:, v:v + 1], bg, H, W)
        assert torch.equal(c1[:, v], c2[:, 0]) and torch.equal(a1[:, v], a2[:, 0]) and torch.equal(r1[:, v], r2[:, 0])
    # 2. deterministic forward
    c3, a3, r3, s3 = raster.forward_raw(g13, vm, pm, bg, H, W)
    assert torch.equal(c1, c3) and torch.equal(a1, a3)
    # 3. ranges: alpha in [0,1), colour = C + T*bg with bg=1 -> within [0, 1+eps]
    assert float(a1[:, :, 1].min()) >= 0.0 and float(a1[:, :, 1].max()) < 1.0
    assert float(c1.min()) >= -1e-5 and float(c1.max()) <= 1.0 + 1e-4
    # 4. every tile list is depth sorted and sum(tile counts) == D
    wsv = raster.workspace_views(s1["ws"], s1["L"], 1, P, V, H, W, s1["max_instances"])
    D = s1["num_rendered"]
    ts = wsv["tile_start"].cpu().numpy().astype(np.int64)
    assert ts[-1] == D
    keys = wsv["keys"][:D].cpu().numpy().view(np.uint64)
    seg = np.zeros(D, dtype=bool); seg[ts[:-1][ts[:-1] < D]] = True
    inc = keys[1:] > keys[:-1]
    assert np.all(inc | seg[1:]), "a tile list is not strictly sorted"
    # 5. one view against the oracle at full size
    o = oracle_view(g, vs[2], ps[2], [1, 1, 1], H, W)
    assert rel_l2(c1[0, 2].cpu().numpy(), o["color"]) <= TOL
    assert np.array_equal(r1[0, 2].cpu().numpy(), o["radii"])
    # 6. backward is linear in the upstream gradient
    torch.manual_seed(0)
    g1 = torch.randn_like(c1); g2 = torch.randn_like(a1)
    ga = raster.backward_raw(s1, g1, g2)
    gb = raster.backward_raw(s1, 2.0 * g1, 2.0 * g2)
    assert rel_l2(gb.cpu().numpy(), 2.0 * ga.cpu().numpy()) <= 1e-4


def test_fused_postprocess_matches_reference_formulas_and_autograd():
    """render_postprocess == the torch ops of /root/reference/nsr/gs_surfel.py:121-163, forward and backward."""
    from gaussiananything_b200 import raster
    dev = torch.device("cuda:0")
    torch.manual_seed(3)
    B, V, H, W = 2, 3, 40, 56
    color = (torch.rand(B, V, 3, H, W, device=dev) * 1.4 - 0.2).requires_grad_(True)       # some values outside [0,1]
    allmap = torch.randn(B, V, 7, H, W, device=dev)
    allmap[0, 0, 5, 0, :5] = float("nan")
    allmap[0, 1, 5, 1, :5] = float("inf")
    allmap = allmap.requires_grad_(True)
    cam = torch.randn(B, V, 4, 4, device=dev)
    outs = raster.render_postprocess(color, allmap, cam)
    ws = [torch.randn_like(o) for o in outs]
    (sum((o * w).sum() for o, w in zip(outs, ws))).backward()
    g_color, g_allmap = color.grad.clone(), allmap.grad.clone()
    color.grad = None; allmap.grad = None
    # reference formulas (per view in the reference, batched here)
    image = color.clamp(0, 1)
    alpha = allmap[:, :, 1:2]
    normal = (allmap[:, :, 2:5].permute(0, 1, 3, 4, 2) @ cam[:, :, None, :3, :3].transpose(-1, -2)).permute(0, 1, 4, 2, 3)
    depth = torch.nan_to_num(allmap[:, :, 5:6], 0, 0)
    dist = allmap[:, :, 6:7]
    refs = (image, alpha, depth, normal, dist)
    for o, r in zip(outs, refs):
        assert o.shape == r.shape and torch.allclose(o, r, atol=1e-5, rtol=1e-5)
    (sum((r * w).sum() for r, w in zip(refs, ws))).backward()
    assert torch.allclose(g_color, color.grad, atol=1e-5)
    fin = torch.isfinite(allmap.detach()[:, :, 5])
    ga_ref = allmap.grad.clone()
    ga_ref[:, :, 5][~fin] = 0.0                      # torch propagates a gradient through nan_to_num; the value is unused
    g_allmap[:, :, 5][~fin] = 0.0
    assert torch.allclose(g_allmap, ga_ref, atol=1e-4, rtol=1e-4)


# ---------------------------------------------------------------------------------------------------------------
# round 2: the reference's own loop as golden, the B3 adapter, C2-size backward, the two switchable judgement calls
# ---------------------------------------------------------------------------------------------------------------
def test_reference_loop_golden():
    """GaussianRenderer2DGS.render (one batched launch set) == the UNMODIFIED /root/reference/nsr/gs_surfel.py
    B x V loop + post-processing, run on CPU over an oracle-backed diff_surfel_rasterization
    (tests/golden/make_gs_surfel_golden.py wrote the fixture)."""
    import os
    from gaussiananything_b200.gs_surfel import GaussianRenderer2DGS
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gs_surfel_loop.npz"))
    dev = torch.device("cuda:0")
    T = lambda a: torch.tensor(a, device=dev)
    r = GaussianRenderer2DGS(64, 3, {"z_near": 0.01})
    tf = float(z["tanfov"])
    a = r.render(T(z["g"]), T(z["view"]), T(z["proj"]), T(z["pos"]), tf)
    b = r.render(T(z["g"][:1]), T(z["view"][:1, :2]), T(z["proj"][:1, :2]), T(z["pos"][:1, :2]), tf,
                 bg_color=T(z["b__bg"]), scale_modifier=1.6, output_size=48)
    for tag, out in (("a", a), ("b", b)):
        assert set(out) == {"image", "alpha", "depth", "rend_normal", "dist"}
        for k, v in out.items():
            want = z["%s__%s" % (tag, k)]
            got = v.cpu().numpy()
            assert got.shape == want.shape, (tag, k, got.shape, want.shape)
            if k == "depth":        # median depth: a pixel whose T crosses 0.5 within rounding picks another surfel
                bad = np.abs(got - want) > 1e-4 * np.maximum(1.0, np.abs(want))
                assert bad.mean() <= 2e-4, (tag, k, bad.mean())
            elif k == "dist":
                assert rel_l2(got, want) <= TOL or np.abs(got - want).max() <= 2e-5, (tag, k)
            else:
                assert rel_l2(got, want) <= TOL, (tag, k, rel_l2(got, want))


def test_gaussian_renderer_render_adapter():
    """Boundary B3: nsr.gaussian_renderer.render(viewpoint_camera, pc, pipe, bg_color, ...) call shape."""
    import math
    from types import SimpleNamespace
    from gaussiananything_b200.gaussian_renderer import render
    P, H = 2500, 112
    g = scene(P, 33, 6.0)
    vs, ps, cs, tf = cameras(1, start=3)
    dev = torch.device("cuda:0")
    gt = torch.tensor(g, device=dev)
    fov = 2.0 * math.atan(tf)
    cam = SimpleNamespace(FoVx=fov, FoVy=fov, image_height=H, image_width=H,
                          world_view_transform=torch.tensor(vs[0], device=dev),
                          full_proj_transform=torch.tensor(ps[0], device=dev),
                          camera_center=torch.tensor(cs[0], device=dev))
    pc = SimpleNamespace(get_xyz=gt[:, 0:3], get_opacity=gt[:, 3:4], get_scaling=gt[:, 4:6], get_rotation=gt[:, 6:10],
                         get_features=gt[:, 10:13], active_sh_degree=0)
    bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
    out = render(cam, pc, SimpleNamespace(debug=False), bg, scaling_modifier=1.3)
    assert {"render", "viewspace_points", "visibility_filter", "radii"} <= set(out)
    o = oracle_view(g, vs[0], ps[0], [0.1, 0.2, 0.3], H, H, scale_modifier=1.3)
    assert rel_l2(out["render"].cpu().numpy(), o["color"]) <= TOL
    assert np.array_equal(out["radii"].cpu().numpy(), o["radii"])
    assert np.array_equal(out["visibility_filter"].cpu().numpy(), o["radii"] > 0)
    out2 = render(cam, pc, SimpleNamespace(debug=False), bg, override_color=torch.flip(gt[:, 10:13], dims=[1]))
    o2 = so_rasterize_colors(g, np.ascontiguousarray(g[:, 10:13][:, ::-1]), vs[0], ps[0], [0.1, 0.2, 0.3], H)
    assert rel_l2(out2["render"].cpu().numpy(), o2["color"]) <= TOL


def so_rasterize_colors(g, colors, view, proj, bg, H):
    from oracle import surfel_oracle as so
    return so.rasterize(g[:, 0:3], g[:, 3:4], g[:, 4:6], g[:, 6:10], colors, view, proj, bg, H, H, 1.0)


def _oracle_grad_sum(g, vs, ps, bg, H, W, gc, ga, views):
    from oracle import surfel_oracle as so
    P = g.shape[0]
    want = np.zeros((P, 13))
    for v in views:
        o = oracle_view(g, vs[v], ps[v], bg, H, W)
        b = so.rasterize_backward(o, gc[v], ga[v])
        want[:, 0:3] += b["means3D"]; want[:, 3:4] += b["opacities"]; want[:, 4:6] += b["scales"]
        want[:, 6:10] += b["rotations"]; want[:, 10:13] += b["colors"]
    return want


GRAD_COLS = [("means3D", slice(0, 3)), ("opacity", slice(3, 4)), ("scales", slice(4, 6)),
             ("rotations", slice(6, 10)), ("colors", slice(10, 13))]


def test_c2_size_backward_vs_oracle():
    """BASELINE configs[1] (100k surfels, 512^2, 6 views): the gradient of the headline workload against the oracle --
    one view alone, and the batched launch's sum over all 6 views."""
    from gaussiananything_b200 import raster
    from oracle import surfel_oracle as so
    import os
    so.set_num_threads(os.cpu_count() or 1)
    P, H, W, V = 100000, 512, 512, 6
    g = scene(P, 40)
    vs, ps, _, _ = cameras(V)
    bg = [1.0, 1.0, 1.0]
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(5)
    gc = rng.standard_normal((V, 3, H, W)).astype(np.float32)
    ga = rng.standard_normal((V, 7, H, W)).astype(np.float32)
    g13 = torch.tensor(g, device=dev)[None]
    bgt = torch.tensor(bg, device=dev)
    # one view
    c, a, r, st = raster.forward_raw(g13, torch.tensor(vs[3:4], device=dev)[None], torch.tensor(ps[3:4], device=dev)[None],
                                     bgt, H, W)
    got1 = raster.backward_raw(st, torch.tensor(gc[3:4], device=dev)[None], torch.tensor(ga[3:4], device=dev)[None])
    want1 = _oracle_grad_sum(g, vs, ps, bg, H, W, gc, ga, [3])
    _check_grad_robust(got1[0].cpu().numpy(), want1, "1 view")
    # all 6 views in one launch set: gradient summed over the views
    c, a, r, st = raster.forward_raw(g13, torch.tensor(vs, device=dev)[None], torch.tensor(ps, device=dev)[None], bgt, H, W)
    got6 = raster.backward_raw(st, torch.tensor(gc, device=dev)[None], torch.tensor(ga, device=dev)[None])
    want6 = _oracle_grad_sum(g, vs, ps, bg, H, W, gc, ga, range(V))
    _check_grad_robust(got6[0].cpu().numpy(), want6, "6 views", worst=6e-4)     # 1e-4 per view


def _check_grad_robust(got, want, tag, worst=1e-4):
    """At 100k sub-pixel surfels a handful of (pixel, surfel) pairs sit within fp32 rounding of a non-differentiable
    decision of the algorithm (rho3d <= rho2d picks the 3-D or the low-pass branch; p.z -> 0); the CUDA path uses
    MUFU reciprocals there, the oracle IEEE divisions, so those pairs can take the other branch and their surfel's
    scale / rotation gradient differs at O(1) (tools/diag_c2_bwd.py: 20 of 100 000 surfels carry the whole excess,
    every column is at 1e-4 without them).  Bar: rel-L2 <= 1e-3 per gradient group once the `worst` fraction of
    surfels (1e-4 = 10 of 100k per view) with the largest error is set aside, and <= 1e-2 with everything in."""
    P = got.shape[0]
    err = np.abs(got - want).sum(1) / (np.abs(want).sum(1) + 1e-3 * np.abs(want).mean())
    keep = np.ones(P, bool)
    keep[np.argsort(-err)[:max(1, int(worst * P))]] = False
    for name, sl in GRAD_COLS:
        r_all, r_keep = rel_l2(got[:, sl], want[:, sl]), rel_l2(got[keep][:, sl], want[keep][:, sl])
        assert r_keep <= TOL, (tag, name, r_keep)
        assert r_all <= 1e-2, (tag, name, r_all)


@pytest.mark.parametrize("radius_formula,quat_norm_grad", [(1, 0), (0, 1), (1, 1)])
def test_switchable_judgement_calls(radius_formula, quat_norm_grad):
    """The two unpinned choices of the restatement (radius formula; quaternion-normalisation gradient) are run-time
    switches in the CUDA path and in the oracle: every combination stays in parity (integers bit-exact), and the
    alternatives really differ from the default."""
    from gaussiananything_b200 import _lib, raster
    from oracle import surfel_oracle as so
    lib = _lib.lib()
    P, H, W = 3000, 96, 112
    g = scene(P, 50, 6.0)
    g[:, 6:10] *= np.linspace(0.5, 2.0, P, dtype=np.float32)[:, None]        # non-unit quaternions
    vs, ps, _, _ = cameras(1, start=2)
    bg = [0.3, 0.6, 0.9]
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(1)
    gc = rng.standard_normal((1, 3, H, W)).astype(np.float32)
    ga = rng.standard_normal((1, 7, H, W)).astype(np.float32)

    def run():
        g13 = torch.tensor(g, device=dev)[None]
        c, a, r, st = raster.forward_raw(g13, torch.tensor(vs, device=dev)[None], torch.tensor(ps, device=dev)[None],
                                         torch.tensor(bg, device=dev), H, W)
        grad = raster.backward_raw(st, torch.tensor(gc, device=dev)[None], torch.tensor(ga, device=dev)[None])
        wsv = raster.workspace_views(st["ws"], st["L"], 1, P, 1, H, W, st["max_instances"])
        return c, a, r, st, wsv, grad[0].cpu().numpy()

    base = run()
    try:
        lib.ga_raster_set_variant(radius_formula, quat_norm_grad)
        so.set_variant(radius_formula, quat_norm_grad)
        c, a, r, st, wsv, grad = run()
        o = oracle_view(g, vs[0], ps[0], bg, H, W)
        assert st["num_rendered"] == o["num_rendered"]
        _check_view(o, c[0, 0], a[0, 0], r[0, 0], wsv, 0, P, H, W)
        want = _oracle_grad_sum(g, vs, ps, bg, H, W, gc, ga, [0])
        for name, sl in GRAD_COLS:
            assert rel_l2(grad[:, sl], want[:, sl]) <= TOL, name
        if radius_formula:
            assert (r[0, 0] >= base[2][0, 0]).all() and (r[0, 0] > base[2][0, 0]).any()
            assert rel_l2(c.cpu().numpy(), base[0].cpu().numpy()) <= 1e-3       # larger tile lists, same pixels
        else:
            assert torch.equal(r, base[2])
        if quat_norm_grad:
            assert rel_l2(grad[:, 6:10], base[5][:, 6:10]) > 1e-2
            q = g[:, 6:10].astype(np.float64)
            assert np.abs((grad[:, 6:10] * q).sum(1)).max() <= 1e-3 * np.abs(grad[:, 6:10]).max() * 4   # radial part removed
    finally:
        lib.ga_raster_set_variant(0, 0)
        so.set_variant(0, 0)


def test_render_sharded_world1_matches_manual_loop():
    """sharding.render_sharded on one rank (no process group) == rendering every (sample, view) pair by hand."""
    from gaussiananything_b200 import sharding
    from gaussiananything_b200.gs_surfel import GaussianRenderer2DGS
    dev = torch.device("cuda:0")
    S, V, P, H = 2, 3, 1500, 64
    g = torch.tensor(np.stack([scene(P, 60, 8.0), scene(P, 61, 5.0)]), device=dev)
    vs, ps, cs, tf = cameras(S * V)
    cv = torch.tensor(vs, device=dev).reshape(S, V, 4, 4)
    cp = torch.tensor(ps, device=dev).reshape(S, V, 4, 4)
    pos = torch.tensor(cs, device=dev).reshape(S, V, 3)
    r = GaussianRenderer2DGS(H, 3, {})
    got = sharding.render_sharded(r, g, cv, cp, pos, tf)
    assert set(got) == {(b, v) for b in range(S) for v in range(V)}
    full = r.render(g, cv, cp, pos, tf)
    for (b, v), d in got.items():
        for k, t in d.items():
            assert torch.equal(t, full[k][b, v]), (b, v, k)


@pytest.mark.parametrize("list_k", [32, 3])
def test_backward_from_recorded_lists_matches_recompute_and_oracle(list_k):
    """list_k > 0: the forward records every pixel's contributions and the backward walks them (no culling, no pair
    re-evaluation).  list_k = 3 overflows in most tiles, which must then take the recompute path: the gradient is
    the same either way (the list path reuses the forward's alpha bits, so not bit-identical) and matches the oracle."""
    from gaussiananything_b200 import raster
    P, H, W, V = 5000, 128, 112, 2
    g = scene(P, 80, 5.0)
    vs, ps, _, _ = cameras(V, start=4)
    bg = [1.0, 0.5, 0.2]
    dev = torch.device("cuda:0")
    g13 = torch.tensor(g, device=dev)[None]
    vm, pm = torch.tensor(vs, device=dev)[None], torch.tensor(ps, device=dev)[None]
    rng = np.random.default_rng(2)
    gc = rng.standard_normal((V, 3, H, W)).astype(np.float32)
    ga = rng.standard_normal((V, 7, H, W)).astype(np.float32)
    dgc, dga = torch.tensor(gc, device=dev)[None], torch.tensor(ga, device=dev)[None]
    c0, a0, r0, s0 = raster.forward_raw(g13, vm, pm, torch.tensor(bg, device=dev), H, W, list_k=0)
    g0 = raster.backward_raw(s0, dgc, dga)[0].cpu().numpy()
    c1, a1, r1, s1 = raster.forward_raw(g13, vm, pm, torch.tensor(bg, device=dev), H, W, list_k=list_k)
    assert torch.equal(c0, c1) and torch.equal(a0, a1)                   # recording does not change the images
    L = s1["L"]
    T = ((W + 15) // 16) * ((H + 15) // 16)
    flags = s1["ws"][L.tile_flag:L.tile_flag + 4 * V * T].view(torch.int32)
    nl = s1["ws"][L.n_list:L.n_list + 4 * V * H * W].view(torch.int32)
    assert int(nl.max()) > 3
    if list_k == 3:
        assert 0 < int(flags.sum()) <= V * T                             # overflowed tiles are flagged ...
    else:
        assert int(flags.sum()) == 0 and int(nl.max()) <= 32
    g1 = raster.backward_raw(s1, dgc, dga)[0].cpu().numpy()
    want = _oracle_grad_sum(g, vs, ps, bg, H, W, gc, ga, range(V))
    for name, sl in GRAD_COLS:
        assert rel_l2(g1[:, sl], want[:, sl]) <= TOL, (name, rel_l2(g1[:, sl], want[:, sl]))
        assert rel_l2(g1[:, sl], g0[:, sl]) <= TOL, name
