"""The forward composite on a scene whose 256-instance chunks need more than one window of its pair buffer, with
surfels whose cull box is unbounded (their box covers every pixel of each tile they touch)."""
import numpy as np
import pytest
import torch

from tests.helpers import cameras, oracle_view, rel_l2, scene

pytestmark = pytest.mark.gpu

FWD_PAIRS = 4096            # csrc/raster_render.cu: pairs per window


def _clipped_pairs(bb, ox, oy, W, H):
    """(instance, pixel) pairs of each cull box clipped to the tile's pixels inside the image, as the kernel counts them."""
    x0 = np.ceil(np.maximum(bb[:, 0], ox)); x1 = np.floor(np.minimum(bb[:, 1], min(ox + 15, W - 1)))
    y0 = np.ceil(np.maximum(bb[:, 2], oy)); y1 = np.floor(np.minimum(bb[:, 3], min(oy + 15, H - 1)))
    return (np.maximum(0, x1 - x0 + 1) * np.maximum(0, y1 - y0 + 1)).astype(np.int64)


def test_forward_multi_window_chunks_keep_state_and_match_oracle():
    from gaussiananything_b200 import raster
    P, H, W, V = 6000, 128, 112, 2
    g = scene(P, 90, 12.0)
    vs, ps, cs, _ = cameras(V, start=7)
    # large opaque surfels just in front of each camera: the cutoff ellipse of some of them reaches the camera plane,
    # and their cull box is unbounded
    rng = np.random.default_rng(1)
    for v in range(V):
        sl = slice(64 * v, 64 * (v + 1))
        ahead = -cs[v] / np.linalg.norm(cs[v])
        g[sl, 0:3] = cs[v] + ahead * rng.uniform(0.3, 0.6, (64, 1)) + rng.uniform(-0.08, 0.08, (64, 3))
        g[sl, 3] = 0.9
        g[sl, 4:6] = 0.2
    bg = [1.0, 0.5, 0.2]
    dev = torch.device("cuda:0")
    g13 = torch.tensor(g, device=dev)[None]
    vm, pm = torch.tensor(vs, device=dev)[None], torch.tensor(ps, device=dev)[None]
    bgt = torch.tensor(bg, device=dev)
    c0, a0, r0, s0 = raster.forward_raw(g13, vm, pm, bgt, H, W, list_k=0)
    w0 = raster.workspace_views(s0["ws"], s0["L"], 1, P, V, H, W, s0["max_instances"])
    nc0 = w0["n_contrib"].clone()
    c1, a1, r1, s1 = raster.forward_raw(g13, vm, pm, bgt, H, W, list_k=32)
    L, ws = s1["L"], s1["ws"]
    w1 = raster.workspace_views(ws, L, 1, P, V, H, W, s1["max_instances"], list_k=32)

    # the scene exercises what it is meant to: unbounded boxes, and chunks cut into several windows
    gx, gy = (W + 15) // 16, (H + 15) // 16
    T = gx * gy
    rec = w1["rec"].cpu().numpy()                                                  # [V, P, 24]
    radii = r1[0].cpu().numpy()
    bbox = rec[:, :, 16:20]
    assert ((bbox[:, :, 0] == np.float32(-1e30)) & (radii > 0)).any(), "no surfel with an unbounded cull box"
    tile_start = w1["tile_start"].cpu().numpy().astype(np.int64)
    ids = w1["ids"].cpu().numpy().astype(np.int64)
    most = 0
    for v in range(V):
        for ty in range(gy):
            for tx in range(gx):
                t = v * T + ty * gx + tx
                sid = ids[tile_start[t]:tile_start[t + 1]]
                pairs = _clipped_pairs(bbox[v, sid], tx * 16, ty * 16, W, H)
                for k in range(0, len(sid), 256):
                    most = max(most, int(pairs[k:k + 256].sum()))
    assert most > 2 * FWD_PAIRS, most

    # recording the lists changes nothing the forward computes
    assert torch.equal(c0, c1) and torch.equal(a0, a1) and torch.equal(r0, r1)
    assert torch.equal(nc0, w1["n_contrib"])                       # last and median contributor
    # the per-instance counts add up to the per-pixel list lengths, tile by tile
    last = w1["n_contrib"][:, 0].cpu().numpy()
    flags = w1["tile_flag"].cpu().numpy()
    n_list = w1["n_list"].cpu().numpy()
    inst_cnt = w1["inst_cnt"].cpu().numpy()
    assert int(n_list.max()) > 3
    for v in range(V):
        for ty in range(gy):
            for tx in range(gx):
                t = v * T + ty * gx + tx
                ys, xs = slice(ty * 16, ty * 16 + 16), slice(tx * 16, tx * 16 + 16)
                assert bool(flags[t]) == bool((n_list[v, ys, xs] > 32).any())
                depth = int(last[v, ys, xs].max())
                got = int(inst_cnt[tile_start[t]:tile_start[t] + depth].astype(np.int64).sum())
                assert got == int(n_list[v, ys, xs].astype(np.int64).sum()), (v, ty, tx)

    for v in range(V):
        o = oracle_view(g, vs[v], ps[v], bg, H, W)
        assert np.array_equal(radii[v], o["radii"])
        assert rel_l2(c1[0, v].cpu().numpy(), o["color"]) <= 1e-3
        a = a1[0, v].cpu().numpy()
        for ch in (0, 1, 2, 3, 4):                 # depth, alpha, normal (median depth and distortion: see test_raster_gpu)
            assert rel_l2(a[ch], o["allmap"][ch]) <= 1e-3, ch
