"""Edge cases of the surfel rasteriser against the fp64 tile walker (tests/raster_ref.py), the C oracle and numpy:
cull-box coverage, the forward's per-pair lists and inst_cnt, the sort and scan boundaries, and per-surfel gradients
with backward chunks of several windows."""
import functools

import numpy as np
import pytest
import torch

from tests import raster_ref as rr
from tests import raster_scenes as rs
from tests.helpers import cameras, oracle_view, rel_l2, scene

pytestmark = pytest.mark.gpu

FWD_PAIRS = 4096            # csrc/raster_render.cu: pairs per forward window
BWD_RECORDS = 4096          # csrc/raster_render.cu: records per backward window
BG = [1.0, 0.5, 0.2]
# Recorded {alpha, depth} of the forward's lists against the fp64 walker, per pair, on the unambiguous part of every
# list.  The kernel is one more binary32 evaluation of each pair (with FMAs and MUFU rcp / ex2), so its error is bounded
# per pair, not by one flat tolerance: on translucent_scene the fp32 error of alpha has a median of 7e-7 and reaches
# 9e-4 on nearly edge-on surfels.
#   alpha: |kernel - fp64| <= LIST_COND_K * alpha_cond, the walker's first-order error bound of any binary32
#          evaluation (median 9e-6 of alpha).  The walker's own two binary32 evaluations reach 0.78 of alpha_cond;
#          the kernel reaches 2.04 of it (H100 80GB HBM3 at 400 W, translucent_scene, 2 views);
#   depth: |kernel - fp64| <= LIST_DEV_K * dev32 + LIST_RTOL * |fp64|, dev32 = the larger deviation of the walker's two
#          binary32 evaluations; the kernel reaches 0.46 of this bound.
LIST_COND_K, LIST_DEV_K, LIST_RTOL = 4.0, 4.0, 1e-5
# Per-pixel bar of the images against the walker on unambiguous pixels: the fp32 C oracle's measured deviation
# (rr.CAL_ORACLE) plus the kernel's MUFU rcp / ex2 (<= 2 ulp per alpha and per 1/depth, i.e. <= 2.4e-7 relative per
# contribution, over at most 256 contributions: 6e-5 of the pixel's magnitude).  Measured on an H100 80GB HBM3 at
# 400 W (translucent_scene, 2 views), per-pixel max-abs per channel (colour 3; depth, alpha, normal 3, median depth,
# distortion): 1.6e-6 2.4e-6 1.7e-6 | 6.2e-6 3.4e-6 4.2e-6 4.6e-6 3.3e-6 9.9e-6 3.3e-7, all below rr.CAL_ORACLE alone.
PIX_ALLOW = 6e-5
# Per-surfel gradient against the C oracle, surfels owning a flagged pair excluded (see _surfel_err).  Measured on an
# H100 80GB HBM3 at 400 W (translucent_scene, 2 views, 2483 of 2500 surfels kept): max 5.0e-4 (list_k 256), 5.1e-4
# (list_k 0 and 8).
GRAD_TOL = 1e-3
# Tiny scene against fp64 autograd of oracle/surfel_torch.py, per gradient group.  Measured on the same H100: rel-L2
# 3.1e-5 (means), 2.4e-6 (opacity), 4.1e-5 (scales), 6.5e-6 (rotations), 2.5e-6 (colours).
TORCH_TOL = 1e-4


def _dev():
    return torch.device("cuda:0")


def _forward(g, vs, ps, H, W, list_k, batch=1, scale_modifier=1.0, bg=BG):
    from gaussiananything_b200 import raster
    dev = _dev()
    P = g.shape[-2]
    V = vs.shape[0] // batch
    g13 = torch.tensor(np.asarray(g, np.float32), device=dev).reshape(batch, P, 13)
    vm = torch.tensor(vs, device=dev).reshape(batch, V, 4, 4)
    pm = torch.tensor(ps, device=dev).reshape(batch, V, 4, 4)
    c, a, r, st = raster.forward_raw(g13, vm, pm, torch.tensor(bg, device=dev), H, W, scale_modifier, list_k=list_k)
    wsv = raster.workspace_views(st["ws"], st["L"], batch, P, V, H, W, st["max_instances"], list_k=list_k)
    return c, a, r, st, {k: v.cpu().numpy() for k, v in wsv.items()}


def _view_order(wsv, v, T):
    ts = wsv["tile_start"].astype(np.int64)[v * T:(v + 1) * T + 1]
    return ts - ts[0], wsv["ids"].astype(np.int64)[ts[0]:ts[-1]]


def _unpack_rect(r):
    r = r.astype(np.int64)
    return np.stack([r & 255, (r >> 8) & 255, (r >> 16) & 255, r >> 24], -1)


# ------------------------------------------------------------------------------------------------ 1. cull box
@pytest.mark.timeout(600)
def test_cull_box_holds_every_clear_pass_pixel():
    """Every pixel where a visible surfel's fp64 alpha is at least (1/255)(1 + 1e-3) lies inside the cull box K1
    computed, and opacity below 1/255 gives the empty box."""
    g, vs, ps, H, W = rs.cull_box_scene()
    SM = rs.CULL_SM
    _, _, radii, _, wsv = _forward(g, vs, ps, H, W, 0, scale_modifier=SM)
    radii = radii[0].cpu().numpy()
    tot = dict(checked=0, bounded=0, unbounded=0, near_edge=0, empty=0, near_switch=0, rect_differs=0, visible=0)
    a255 = np.float32(1) / np.float32(255)
    for v in range(vs.shape[0]):
        ratio, geo = rs._switch_ratio(g, vs[v], ps[v], H, W)
        bb = wsv["rec"][v, :, 16:20].astype(np.float64)
        low = (g[:, 3] < a255) & (radii[v] > 0)
        assert np.all(bb[low] == np.array([1e30, -1e30, 1e30, -1e30], np.float32)), "opacity < 1/255, non-empty box"
        tot["empty"] += int(low.sum())
        # surfels whose fp64 tile rectangle is the kernel's (a few adversarial ones round differently)
        use = (radii[v] > 0) & (geo["radii"] > 0) & np.all(_unpack_rect(wsv["rect"][v]) == geo["rect"], 1)
        tot["visible"] += int((radii[v] > 0).sum())
        tot["rect_differs"] += int(((radii[v] > 0) & ~use).sum())
        cnt, x0, x1, y0, y1 = rr.clear_pass_boxes(geo)
        use &= cnt > 0
        inside = (x0 >= bb[:, 0]) & (x1 <= bb[:, 1]) & (y0 >= bb[:, 2]) & (y1 <= bb[:, 3])
        bad = np.nonzero(use & ~inside)[0]
        assert bad.size == 0, ("clear-pass pixels outside the cull box", v, bad[:10].tolist(),
                               [(bb[i].tolist(), [x0[i], x1[i], y0[i], y1[i]]) for i in bad[:3]])
        bounded = use & (np.abs(bb[:, 0]) < 1e29)
        tot["checked"] += int(use.sum())
        tot["bounded"] += int(bounded.sum())
        tot["near_switch"] += int((bounded & (ratio >= -1e-2) & (ratio < -1e-3)).sum())   # within a decade of it
        tot["unbounded"] += int((use & (bb[:, 0] == float(np.float32(-1e30)))).sum())     # K1's unbounded branch
        gap = np.minimum(np.minimum(x0 - bb[:, 0], bb[:, 1] - x1), np.minimum(y0 - bb[:, 2], bb[:, 3] - y1))
        tot["near_edge"] += int((bounded & (gap <= 1.0)).sum())
    print("cull box:", tot)
    assert tot["bounded"] > 0 and tot["unbounded"] > 0 and tot["near_edge"] > 0 and tot["empty"] > 0, tot
    # the switch: bounded boxes with dt / Tw_z^2 in [-1e-2, -1e-3) (1157 clear-pass surfels there in view 0, fp64)
    assert tot["near_switch"] >= 800, tot
    # surfels whose fp64 radius or tile rectangle rounds differently from the kernel's are left out: few of them
    assert tot["rect_differs"] <= 0.02 * tot["visible"], tot


# ------------------------------------------------------------------------------------------------ 2. pair lists
@functools.lru_cache(maxsize=None)
def _translucent(list_k):
    g, vs, ps, H, W = rs.translucent_scene()
    c, a, r, st, wsv = _forward(g, vs, ps, H, W, list_k)
    T = ((W + 15) // 16) * ((H + 15) // 16)
    walks = [rr.walk(rr.geometry(g, vs[v], ps[v], H, W), *_view_order(wsv, v, T), BG) for v in range(vs.shape[0])]
    return g, vs, ps, H, W, c.cpu().numpy(), a.cpu().numpy(), st, wsv, walks


def _clipped_pairs(bb, ox, oy, W, H):
    x0 = np.ceil(np.maximum(bb[:, 0], ox)); x1 = np.floor(np.minimum(bb[:, 1], min(ox + 15, W - 1)))
    y0 = np.ceil(np.maximum(bb[:, 2], oy)); y1 = np.floor(np.minimum(bb[:, 3], min(oy + 15, H - 1)))
    return (np.maximum(0, x1 - x0 + 1) * np.maximum(0, y1 - y0 + 1)).astype(np.int64)


@pytest.mark.timeout(600)
def test_forward_pair_lists_match_fp64_walker():
    """list_k = 256 (nothing overflows): every pixel's recorded list against the walker's contributions."""
    K = 256
    g, vs, ps, H, W, color, allmap, st, wsv, walks = _translucent(K)
    V = vs.shape[0]
    gx, gy = (W + 15) // 16, (H + 15) // 16
    T = gx * gy
    assert wsv["tile_flag"].sum() == 0 and wsv["n_list"].max() <= K
    ts_all = wsv["tile_start"].astype(np.int64)
    ids_all = wsv["ids"].astype(np.int64)
    pix_tile = (np.arange(H)[:, None] // 16) * gx + np.arange(W)[None] // 16               # [H, W]
    pix_loc = (np.arange(H)[:, None] % 16) * 16 + np.arange(W)[None] % 16
    most_pairs, straddle, amb_total, rt_a, rt_d, dev, bars = 0, 0, 0, 0.0, 0.0, np.zeros(10), np.zeros(10)
    med_a = 0.0
    for v in range(V):
        w = walks[v]
        lists = wsv["lists"][v * T:(v + 1) * T]                                            # [T, K, 256, 4]
        kl = lists[pix_tile.ravel(), :, pix_loc.ravel(), :]                                # [HW, K, 4]
        nl = wsv["n_list"][v].ravel()
        kpos = np.where(np.arange(K)[None] < nl[:, None], kl[:, :, 0].astype(np.int64), -1)
        kalpha, kdepth = kl[:, :, 1].view(np.float32), kl[:, :, 2].view(np.float32)
        # the walker's contributions as the same [HW, K] table
        pr = w["pairs"]
        start = np.searchsorted(pr["pix"], np.arange(H * W))
        rank = np.arange(pr["pix"].size) - start[pr["pix"]]
        assert rank.max() < K
        wpos = np.full((H * W, K), -1, np.int64); wal = np.zeros((H * W, K)); wde = np.zeros((H * W, K))
        wpos[pr["pix"], rank] = pr["pos"]; wal[pr["pix"], rank] = pr["alpha"]; wde[pr["pix"], rank] = pr["depth"]
        wal_c = np.zeros((H * W, K)); wde_d = np.zeros((H * W, K))
        wal_c[pr["pix"], rank] = pr["alpha_cond"]; wde_d[pr["pix"], rank] = pr["depth_dev32"]
        amb = w["ambiguous"].ravel()
        amb_from = w["amb_from"].ravel()[:, None]
        amb_total += int(amb.sum())
        # position sequences: equal on unambiguous pixels, equal up to the first flagged pair elsewhere
        assert np.array_equal(np.where(kpos < amb_from, kpos, -1), np.where(wpos < amb_from, wpos, -1)), v
        un = ~amb
        assert np.array_equal(nl[un], w["n_list"].ravel()[un])
        nc = wsv["n_contrib"][v]
        assert np.array_equal(nc[0][~w["ambiguous"]], w["last"][~w["ambiguous"]])
        assert np.array_equal(nc[1][~w["ambiguous"]], w["median"][~w["ambiguous"]])
        both = (kpos >= 0) & (kpos < amb_from)
        # per pair: deviation over its bound (<= 1 passes)
        rt_a = max(rt_a, float((np.abs(kalpha - wal) / (LIST_COND_K * wal_c))[both].max()))
        rt_d = max(rt_d, float((np.abs(kdepth - wde) / (LIST_DEV_K * wde_d + LIST_RTOL * wde))[both].max()))
        med_a = max(med_a, float(np.median((np.abs(kalpha - wal) / wal)[both])))
        # inst_cnt, per instance: the number of this view's pixel lists holding the position
        ts = ts_all[v * T:(v + 1) * T + 1]
        per = np.zeros(ts_all[-1], np.int64)
        tt = np.broadcast_to(pix_tile.ravel()[:, None], kpos.shape)
        ok = kpos >= 0
        np.add.at(per, ts[tt[ok]] + kpos[ok], 1)
        last = nc[0]
        for t in range(T):
            ty, tx = divmod(t, gx)
            deep = int(last[ty * 16:ty * 16 + 16, tx * 16:tx * 16 + 16].max())
            assert np.array_equal(wsv["inst_cnt"][ts[t]:ts[t] + deep], per[ts[t]:ts[t] + deep]), (v, t)
            pos_t = kpos[(tt == t) & ok]
            straddle += bool((pos_t < 256).any() and (pos_t >= 256).any())
            sid = ids_all[ts[t]:ts[t + 1]]
            pairs = _clipped_pairs(wsv["rec"][v, sid, 16:20].astype(np.float64), tx * 16, ty * 16, W, H)
            for k in range(0, len(sid), 256):
                most_pairs = max(most_pairs, int(pairs[k:k + 256].sum()))
        # images on unambiguous pixels, per pixel, against the walker
        for ch, (got, want) in enumerate([(color[0, v, c], w["color"][c]) for c in range(3)] +
                                         [(allmap[0, v, c], w["allmap"][c]) for c in range(7)]):
            d = float(np.abs(got - want)[~w["ambiguous"]].max())
            dev[ch] = max(dev[ch], d)
            bars[ch] = max(bars[ch], rr.CAL_ORACLE[ch] + PIX_ALLOW * max(1.0, float(np.abs(want).max())))
    print("pair lists: most pairs per chunk %d, tiles straddling a chunk %d, ambiguous pixels %d of %d, "
          "alpha / bound max %.2f (median relative error %.1e), depth / bound max %.2f, per-pixel max-abs %s" % (
              most_pairs, straddle, amb_total, V * H * W, rt_a, med_a, rt_d, np.array2string(dev, precision=2)))
    assert most_pairs > 2 * FWD_PAIRS, most_pairs          # some chunk needs >= 3 windows
    assert straddle > 0
    assert rt_a <= 1.0 and rt_d <= 1.0, (rt_a, rt_d)
    assert np.all(dev <= bars), (dev, bars)
    assert amb_total <= 0.005 * V * H * W, amb_total


# ------------------------------------------------------------------------------------------------ 3. sort / scan
def _identity_camera(W, H, tanfov=0.5):
    n, f = 0.01, 100.0
    Pm = np.zeros((4, 4), np.float32)
    Pm[0, 0] = Pm[1, 1] = 1.0 / tanfov
    Pm[3, 2] = 1.0
    Pm[2, 2] = f / (f - n)
    Pm[2, 3] = -(f * n) / (f - n)
    return np.eye(4, dtype=np.float32), np.ascontiguousarray(Pm.T)


def _one_tile_surfels(counts, W, H, seed, tanfov=0.5):
    """Tiny surfels centred at pixel (8, 8) of their tile (radius 3: exactly one tile each), counts[t] in tile t, ids
    shuffled over the tiles, view depths drawn from a few values so that many depth keys tie."""
    rng = np.random.default_rng(seed)
    gx = (W + 15) // 16
    tile = np.repeat(np.arange(len(counts)), counts)
    rng.shuffle(tile)
    P = tile.size
    z = np.where(rng.uniform(size=P) < 0.7, rng.choice([1.0, 1.25, 2.0], P), rng.uniform(0.8, 3.0, P))
    px = (tile % gx) * 16 + 8.0
    py = (tile // gx) * 16 + 8.0
    g = np.zeros((P, 13), np.float32)
    g[:, 0] = (px - (W - 1) / 2) * 2 * tanfov * z / W
    g[:, 1] = (py - (H - 1) / 2) * 2 * tanfov * z / H
    g[:, 2] = z
    g[:, 3] = rng.uniform(0.05, 0.9, P)
    g[:, 4:6] = 1e-5
    g[:, 6] = 1.0
    g[:, 10:13] = rng.uniform(0, 1, (P, 3))
    return g, tile


def _numpy_sort(wsv, NV, T, P, gx):
    """tile_start, keys, ids and per-tile counts from the rectangles and depths read back: lexsort of (tile, depth
    bits, surfel id)."""
    rect = _unpack_rect(wsv["rect"].reshape(NV, P))
    dbits = wsv["depth"].reshape(NV, P).view(np.uint32).astype(np.uint64)
    v_i, i_i = np.nonzero(wsv["rect"].reshape(NV, P) != 0)
    tiles, ids = [], []
    for v, i in zip(v_i, i_i):
        x0, y0, x1, y1 = rect[v, i]
        tt = (np.arange(y0, y1)[:, None] * gx + np.arange(x0, x1)[None]).ravel()
        tiles.append(v * T + tt); ids.append(np.full(tt.size, i));
    tiles = np.concatenate(tiles); ids = np.concatenate(ids)
    vv = tiles // T
    kd = dbits[vv, ids]
    o = np.lexsort((ids, kd, tiles))
    tiles, ids, kd = tiles[o], ids[o], kd[o]
    cnt = np.bincount(tiles, minlength=NV * T)
    ts = np.concatenate([[0], np.cumsum(cnt)])
    return ts, (kd << np.uint64(32)) | ids.astype(np.uint64), ids, cnt


def _assert_sorted_like_numpy(wsv, NV, T, P, gx):
    ts, keys, ids, cnt = _numpy_sort(wsv, NV, T, P, gx)
    D = int(ts[-1])
    assert np.array_equal(wsv["tile_start"].astype(np.int64), ts), "tile_start"
    assert np.array_equal(wsv["keys"][:D].view(np.uint64), keys), "keys"
    assert np.array_equal(wsv["ids"][:D].astype(np.int64), ids), "ids"
    st = wsv["status"]
    assert st[0] == D and st[2] == int((cnt > 4096).sum()) and st[3] == int((cnt > 512).sum()), (st[:4].tolist(),)
    assert set(wsv["big_tiles"][:st[3]].tolist()) == set(np.nonzero(cnt > 512)[0].tolist())
    return cnt


@pytest.mark.timeout(600)
def test_sort_boundaries_and_depth_ties():
    counts = [0, 1, 2, 31, 32, 33, 127, 128, 129, 255, 256, 257, 511, 512, 513, 4095, 4096, 4097, 9000, 0]
    perm = np.random.default_rng(3).permutation(len(counts))
    counts = [counts[i] for i in perm]
    W, H = 80, 64
    g, tile = _one_tile_surfels(counts, W, H, seed=1)
    vm, pm = _identity_camera(W, H)
    P = g.shape[0]
    c, a, r, st, wsv = _forward(g, vm[None], pm[None], H, W, 0, bg=[1.0, 1.0, 1.0])
    rect = _unpack_rect(wsv["rect"][0])
    gx = W // 16
    assert np.array_equal(rect[:, 0], tile % gx) and np.array_equal(rect[:, 2], tile % gx + 1)
    assert np.array_equal(rect[:, 1], tile // gx) and np.array_equal(rect[:, 3], tile // gx + 1)
    assert np.all(r.cpu().numpy() == 3)
    cnt = _assert_sorted_like_numpy(wsv, 1, gx * (H // 16), P, gx)
    assert np.array_equal(cnt, np.array(counts))
    dk = wsv["keys"][:int(wsv["status"][0])].view(np.uint64) >> np.uint64(32)
    assert (dk[1:] == dk[:-1]).sum() > 1000                        # depth ties, ordered by id
    o = oracle_view(g, vm, pm, [1.0, 1.0, 1.0], H, W)
    assert np.array_equal(wsv["ids"][:o["num_rendered"]], o["ids"])
    assert np.array_equal(wsv["n_contrib"][0], o["n_contrib"])
    assert rel_l2(c[0, 0].cpu().numpy(), o["color"]) <= 1e-5 and rel_l2(a[0, 0].cpu().numpy(), o["allmap"]) <= 1e-5


@pytest.mark.timeout(600)
def test_sort_more_big_tiles_than_ctas():
    """2 x SM-count tiles above 512 instances, exactly one of them above 4096: every big-tile CTA sorts two tiles, so
    the CTA holding the large tile also sorts one in shared memory.  That mixture holds by construction of the scene;
    what the test checks is that the listing and the sorted result are right when a CTA reuses s_keys and changes
    path between its tiles."""
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    nbig = 2 * nsm
    W = 256
    H = 16 * ((nbig + 8 + 15) // 16)
    T = (W // 16) * (H // 16)
    rng = np.random.default_rng(7)
    counts = np.zeros(T, np.int64)
    big = rng.choice(T, nbig, replace=False)
    counts[big] = rng.integers(513, 700, nbig)
    counts[big[0]] = 4100
    small = np.setdiff1d(np.arange(T), big)
    counts[small] = rng.integers(0, 300, small.size)
    g, _ = _one_tile_surfels(counts.tolist(), W, H, seed=2)
    vm, pm = _identity_camera(W, H)
    c, a, r, st, wsv = _forward(g, vm[None], pm[None], H, W, 0)
    cnt = _assert_sorted_like_numpy(wsv, 1, T, g.shape[0], W // 16)
    assert np.array_equal(cnt, counts)
    big_ctas = min(T, nsm)
    bt = wsv["big_tiles"][:int(wsv["status"][3])]
    assert bt.size == 2 * big_ctas
    large = cnt[bt] > 4096
    assert (large[:big_ctas] != large[big_ctas:]).any(), "no CTA sorted both a shared- and a global-memory tile"


@pytest.mark.timeout(900)
@pytest.mark.parametrize("B,V,H,W", [(2, 5, 512, 512), (1, 8, 656, 400)])
def test_tile_scan_second_pass(B, V, H, W):
    """NV * T above the 8192 tiles one pass of the scan covers: 10 240 tiles, and 8 200 just above."""
    T = ((W + 15) // 16) * ((H + 15) // 16)
    assert B * V * T > 8192
    P = 20000
    g = np.stack([scene(P, 900 + b, 2.0) for b in range(B)])
    vs, ps, _, _ = cameras(B * V, start=3)
    c, a, r, st, wsv = _forward(g, vs, ps, H, W, 0, batch=B)
    _assert_sorted_like_numpy(wsv, B * V, T, P, (W + 15) // 16)
    for nv in range(B * V):
        b, v = divmod(nv, V)
        c1, a1, r1, _, _ = _forward(g[b], vs[nv:nv + 1], ps[nv:nv + 1], H, W, 0)
        assert torch.equal(c[b, v], c1[0, 0]) and torch.equal(a[b, v], a1[0, 0]) and torch.equal(r[b, v], r1[0, 0]), nv
    o = oracle_view(g[B - 1], vs[-1], ps[-1], BG, H, W)
    assert rel_l2(c[B - 1, V - 1].cpu().numpy(), o["color"]) <= 1e-3


# ------------------------------------------------------------------------------------------------ 4. backward
def _surfel_err(got, want):
    """Per surfel: L1 error over its 13 gradient components relative to its L1 norm, floored at 1e-3 of the mean."""
    n = np.abs(want).sum(1)
    return np.abs(got - want).sum(1) / (n + 1e-3 * n.mean())


@pytest.mark.timeout(900)
@pytest.mark.parametrize("list_k", [256, 0, 8])
def test_backward_per_surfel_gradients(list_k):
    """Backward chunks of more than 4096 records (several windows) and tiles above 256 instances; the gradient of
    every surfel that owns no flagged pair matches the C oracle."""
    from gaussiananything_b200 import raster
    from oracle import surfel_oracle as so
    g, vs, ps, H, W, _, _, _, wsv256, walks = _translucent(256)
    V, P = vs.shape[0], g.shape[0]
    T = ((W + 15) // 16) * ((H + 15) // 16)
    gx = (W + 15) // 16
    # records per backward chunk, from the forward's exact counts
    ts_all = wsv256["tile_start"].astype(np.int64)
    most = 0
    for t in range(V * T):
        v, tl = divmod(t, T)
        ty, tx = divmod(tl, gx)
        hi = int(wsv256["n_contrib"][v, 0, ty * 16:ty * 16 + 16, tx * 16:tx * 16 + 16].max())
        ic = wsv256["inst_cnt"][ts_all[t]:ts_all[t] + hi].astype(np.int64)
        for h in range(hi, 0, -256):
            most = max(most, int(ic[max(0, h - 256):h].sum()))
    assert most > BWD_RECORDS, most
    assert (np.diff(ts_all) > 256).any()
    c, a, r, st, wsv = _forward(g, vs, ps, H, W, list_k)
    if list_k == 8:
        fl = wsv["tile_flag"]
        assert fl.any() and not fl.all()
    rng = np.random.default_rng(11)
    gc = rng.standard_normal((V, 3, H, W)).astype(np.float32)
    ga = rng.standard_normal((V, 7, H, W)).astype(np.float32)
    dev = _dev()
    got = raster.backward_raw(st, torch.tensor(gc, device=dev)[None], torch.tensor(ga, device=dev)[None])[0]
    got = got.cpu().numpy().astype(np.float64)
    want = np.zeros((P, 13))
    for v in range(V):
        o = oracle_view(g, vs[v], ps[v], BG, H, W)
        b = so.rasterize_backward(o, gc[v], ga[v])
        want += np.concatenate([b["means3D"], b["opacities"], b["scales"], b["rotations"], b["colors"]], 1)
    keep = np.ones(P, bool)
    for w in walks:
        keep[w["flagged_ids"]] = False
    err = _surfel_err(got, want)
    print("list_k %d: backward chunk records %d, surfels kept %d of %d, per-surfel error max %.2e (all: %.2e)" %
          (list_k, most, keep.sum(), P, err[keep].max(), err.max()))
    assert keep.sum() >= 0.9 * P
    assert err[keep].max() <= GRAD_TOL, (np.argsort(-err * keep)[:5], np.sort(err[keep])[-5:])


@pytest.mark.timeout(300)
def test_tiny_scene_gradient_matches_fp64_autograd():
    from gaussiananything_b200 import raster
    from oracle import surfel_torch as st_
    g, vs, ps, H, W = rs.tiny_scene()
    P = g.shape[0]
    dev = _dev()
    rng = np.random.default_rng(4)
    gc = rng.standard_normal((3, H, W)); ga = rng.standard_normal((7, H, W))
    g13 = torch.tensor(g, device=dev)[None].requires_grad_(True)
    color, allmap, _ = raster.rasterize_surfels_batched(g13, torch.tensor(vs, device=dev)[None],
                                                        torch.tensor(ps, device=dev)[None], torch.tensor(BG, device=dev),
                                                        H, W, 1.0)
    ((color[0, 0] * torch.tensor(gc, device=dev, dtype=torch.float32)).sum() +
     (allmap[0, 0] * torch.tensor(ga, device=dev, dtype=torch.float32)).sum()).backward()
    got = g13.grad[0].cpu().numpy().astype(np.float64)
    t = torch.tensor(g, dtype=torch.float64, requires_grad=True)
    c64, _, a64 = st_.rasterize(t[:, 0:3], t[:, 3:4], t[:, 4:6], t[:, 6:10], t[:, 10:13], torch.tensor(vs[0]),
                                torch.tensor(ps[0]), torch.tensor(BG, dtype=torch.float64), H, W)
    ((c64 * torch.tensor(gc)).sum() + (a64 * torch.tensor(ga)).sum()).backward()
    want = t.grad.numpy()
    errs = {name: rel_l2(got[:, sl], want[:, sl]) for name, sl in
            [("means3D", slice(0, 3)), ("opacity", slice(3, 4)), ("scales", slice(4, 6)), ("rotations", slice(6, 10)),
             ("colors", slice(10, 13))]}
    print("tiny scene vs fp64 autograd:", {k: "%.2e" % e for k, e in errs.items()})
    assert rel_l2(color[0, 0].detach().cpu().numpy(), c64.detach().numpy()) <= 1e-5
    for k, e in errs.items():
        assert e <= TORCH_TOL, (k, e)
