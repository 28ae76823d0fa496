"""Self-checks of the fp64 tile walker (tests/raster_ref.py): against the fp32 C oracle and against fp64 autograd of
oracle/surfel_torch.py.  Host only."""
import numpy as np
import pytest
import torch

from tests import raster_ref as rr
from tests import raster_scenes as rs
from tests.helpers import cameras, oracle_view, scene

BG = [1.0, 0.5, 0.2]


def _oracle_order(o):
    rg = o["ranges"].astype(np.int64)
    ts = np.zeros(len(rg) + 1, np.int64)
    ts[1:] = np.cumsum(rg[:, 1] - rg[:, 0])
    return ts, o["ids"].astype(np.int64)


@pytest.mark.parametrize("P,H,W,boost,seed", [(3000, 128, 112, 8.0, 1), (500, 64, 48, 40.0, 2), (4000, 128, 128, 1.0, 4)])
def test_geometry_and_binning_match_c_oracle(P, H, W, boost, seed):
    g = scene(P, seed, boost)
    vs, ps, _, _ = cameras(1, start=seed)
    o = oracle_view(g, vs[0], ps[0], BG, H, W)
    geo = rr.geometry(g, vs[0], ps[0], H, W)
    assert np.array_equal(geo["radii"], o["radii"])
    vis = o["radii"] > 0
    assert np.array_equal(geo["rect"][vis], o["rect"][vis])
    ts, ids = rr.bin_tiles(geo)
    assert np.array_equal(ids, o["ids"])
    assert np.array_equal((ts, ids)[0], _oracle_order(o)[0])
    w = rr.walk(geo, ts, ids, BG)
    un = ~w["ambiguous"]
    assert un.mean() >= 0.999
    assert np.array_equal(w["last"][un], o["n_contrib"][0][un])
    assert np.array_equal(w["median"][un], o["n_contrib"][1][un])
    want = np.concatenate([o["color"], o["allmap"]])
    dev = np.abs(np.concatenate([w["color"], w["allmap"]]) - want)[:, un].max(1)
    # measured on the host: 1.1e-4 abs on the depth channel of the first scene (values up to about 3), below 4e-5 elsewhere
    assert np.all(dev <= 1e-4 * np.maximum(1.0, np.abs(want).reshape(10, -1).max(1))), dev
    assert w["pairs"]["pos"].size == int(w["n_list"].sum())


def test_walker_matches_fp64_autograd_forward():
    """The walker and oracle/surfel_torch.py state the same forward: in fp64 they agree to rounding."""
    from oracle import surfel_torch as st
    g, vs, ps, H, W = rs.tiny_scene()
    geo = rr.geometry(g, vs[0], ps[0], H, W)
    w = rr.walk(geo, *rr.bin_tiles(geo), BG)
    t = torch.tensor(g, dtype=torch.float64)
    c, radii, a = st.rasterize(t[:, 0:3], t[:, 3:4], t[:, 4:6], t[:, 6:10], t[:, 10:13], torch.tensor(vs[0]),
                               torch.tensor(ps[0]), torch.tensor(BG, dtype=torch.float64), H, W)
    assert np.array_equal(radii.numpy(), geo["radii"])
    assert np.abs(c.numpy() - w["color"]).max() <= 1e-12
    assert np.abs(a.numpy() - w["allmap"]).max() <= 1e-12
    assert w["n_list"].max() > 1


def test_calibration_against_c_oracle():
    """Per-pixel max-abs deviation of the fp32 C oracle from the walker on unambiguous pixels, over the scenes of
    tests/raster_scenes.py (cull-box scene at scale_modifier 1.3 and 3 views, translucent scene 2 views, tiny scene),
    walking the oracle's own tile order.  Measured on the host, per channel (colour 3; depth, alpha, normal 3, median
    depth, distortion):
        1.4e-5 8.1e-6 8.7e-6 | 5.2e-6 2.9e-6 3.6e-5 1.9e-5 3.5e-5 5.4e-6 2.6e-6
    with 42 ambiguous pixels out of 62 496.  rr.CAL_ORACLE holds these rounded up; last and median contributor
    agree on every unambiguous pixel."""
    dev = np.zeros(10)
    amb = 0
    for fn, sm in ((rs.cull_box_scene, rs.CULL_SM), (rs.translucent_scene, 1.0), (rs.tiny_scene, 1.0)):
        g, vs, ps, H, W = fn()
        for v in range(vs.shape[0]):
            o = oracle_view(g, vs[v], ps[v], BG, H, W, sm)
            w = rr.walk(rr.geometry(g, vs[v], ps[v], H, W, sm), *_oracle_order(o), BG)
            un = ~w["ambiguous"]
            amb += int((~un).sum())
            assert np.array_equal(w["last"][un], o["n_contrib"][0][un])
            assert np.array_equal(w["median"][un], o["n_contrib"][1][un])
            d = np.concatenate([np.abs(w["color"] - o["color"]), np.abs(w["allmap"] - o["allmap"])])[:, un].max(1)
            dev = np.maximum(dev, d)
    print("C oracle vs walker, per-pixel max-abs:", np.array2string(dev, precision=2), "ambiguous pixels", amb)
    assert np.all(dev <= np.array(rr.CAL_ORACLE)), dev
    assert 0 < amb <= 100


def test_flags_mark_a_pair_at_the_alpha_threshold():
    """A surfel whose fp64 alpha at a pixel sits at 1/255 within the margin is flagged, and the pixel is ambiguous."""
    g, vs, ps, H, W = rs.tiny_scene()
    geo = rr.geometry(g[:1], vs[0], ps[0], H, W)
    i = 0
    assert geo["radii"][i] > 0
    x, y = int(round(geo["cx"][i])), int(round(geo["cy"][i]))
    r, _, _ = rr._pairs(geo, np.array([i]), np.array([float(x)]), np.array([float(y)]), x - x % 16, y - y % 16)
    g2 = g[:1].copy()
    g2[0, 3] = np.float32((1.0 / 255.0) * (g[0, 3] / r["alpha"][0, 0]))          # alpha(x, y) == 1/255
    geo2 = rr.geometry(g2, vs[0], ps[0], H, W)
    w = rr.walk(geo2, *rr.bin_tiles(geo2), BG)
    assert w["ambiguous"][y, x] and 0 in w["flagged_ids"]
