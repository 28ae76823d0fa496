"""The backward's per-surfel gradient rows on the GPU: render_bwd applies each view's chain rule to every (tile,
instance) partial sum and adds it to one 16-float row per (batch item, surfel); preprocess_bwd finishes from that row.
Checked against the fp64 oracle where the rows see every case the per-view chain rule has: surfels that only some
views see, the low-pass (mean-2D) branch, back-facing surfels, tiles that take the recompute path, and both
quaternion-gradient variants."""
import numpy as np
import pytest
import torch

from tests.helpers import cameras, oracle_view, rel_l2, scene

pytestmark = pytest.mark.gpu

TOL = 1e-3
GRAD_COLS = [("means3D", slice(0, 3)), ("opacity", slice(3, 4)), ("scales", slice(4, 6)),
             ("rotations", slice(6, 10)), ("colors", slice(10, 13))]
B, V, P, H, W = 2, 3, 2500, 112, 96


def _scene():
    # item 0: the default size mix (mostly small surfels, many of them on the low-pass branch); item 1: larger ones.
    # A fifth of every item sits far to one side, where only some of the orbit cameras see it.
    g = np.stack([scene(P, 90), scene(P, 91, 6.0)])
    g[:, : P // 5, 0] += 0.9
    return g


def _inputs(dev):
    g = _scene()
    vs, ps, _, _ = cameras(B * V, start=1)
    rng = np.random.default_rng(7)
    gc = rng.standard_normal((B * V, 3, H, W)).astype(np.float32)
    ga = rng.standard_normal((B * V, 7, H, W)).astype(np.float32)
    t = dict(g13=torch.tensor(g, device=dev), vm=torch.tensor(vs, device=dev).reshape(B, V, 4, 4),
             pm=torch.tensor(ps, device=dev).reshape(B, V, 4, 4), bg=torch.tensor([1.0, 0.5, 0.2], device=dev),
             gc=torch.tensor(gc, device=dev).reshape(B, V, 3, H, W),
             ga=torch.tensor(ga, device=dev).reshape(B, V, 7, H, W))
    return g, vs, ps, gc, ga, t


def _oracle(g, vs, ps, gc, ga):
    from oracle import surfel_oracle as so
    want = np.zeros((B, P, 13))
    mean2d = np.zeros((B, P))
    for b in range(B):
        for v in range(V):
            nv = b * V + v
            o = oracle_view(g[b], vs[nv], ps[nv], [1.0, 0.5, 0.2], H, W)
            r = so.rasterize_backward(o, gc[nv], ga[nv])
            want[b, :, 0:3] += r["means3D"]; want[b, :, 3:4] += r["opacities"]; want[b, :, 4:6] += r["scales"]
            want[b, :, 6:10] += r["rotations"]; want[b, :, 10:13] += r["colors"]
            mean2d[b] += np.abs(r["dL_dmean2D"]).sum(1)
    return want, mean2d


@pytest.mark.parametrize("list_k,quat_norm_grad", [(32, 0), (32, 1), (3, 0), (3, 1)])
def test_grad_rows_match_oracle(list_k, quat_norm_grad):
    from gaussiananything_b200 import _lib, raster
    from oracle import surfel_oracle as so
    dev = torch.device("cuda:0")
    g, vs, ps, gc, ga, t = _inputs(dev)
    try:
        _lib.lib().ga_raster_set_variant(0, quat_norm_grad)
        so.set_variant(0, quat_norm_grad)
        _, _, radii, st = raster.forward_raw(t["g13"], t["vm"], t["pm"], t["bg"], H, W, list_k=list_k)
        got = raster.backward_raw(st, t["gc"], t["ga"]).cpu().numpy().astype(np.float64)
        want, mean2d = _oracle(g, vs, ps, gc, ga)
    finally:
        _lib.lib().ga_raster_set_variant(0, 0)
        so.set_variant(0, 0)
    # the cases are present: surfels seen in only some views, the low-pass branch, both normal signs, recompute tiles
    seen = (radii.cpu().numpy() > 0)                                            # [B, V, P]
    assert (seen.any(1) & ~seen.all(1)).sum() >= 50
    assert (mean2d > 0).sum() >= 100
    wsv = raster.workspace_views(st["ws"], st["L"], B, P, V, H, W, st["max_instances"], list_k=list_k)
    sign = wsv["rec"][:, :, 22].cpu().numpy().reshape(B, V, P)[seen]
    assert set(np.unique(sign)) == {-1.0, 1.0}
    n_flagged = int(wsv["tile_flag"].sum())
    assert (n_flagged > 0) if list_k == 3 else (n_flagged == 0)
    for b in range(B):
        for name, sl in GRAD_COLS:
            r = rel_l2(got[b][:, sl], want[b][:, sl])
            assert r <= TOL, (b, name, r)


def test_oversized_scratch_with_garbage_gives_the_same_grad():
    """Only the leading batch*P*16 floats of the scratch are zeroed and used: a larger buffer full of garbage gives the
    same gradient, and the bytes after the rows stay as they were."""
    from gaussiananything_b200 import _lib, raster
    from gaussiananything_b200._launch import ptr, stream
    dev = torch.device("cuda:0")
    g, vs, ps, gc, ga, t = _inputs(dev)
    _, _, _, st = raster.forward_raw(t["g13"], t["vm"], t["pm"], t["bg"], H, W, list_k=32)
    lib = _lib.lib()

    def run(scratch):
        grad = torch.empty(B, P, 13, device=dev)
        _lib.check(lib.ga_raster_backward_ex(
            ptr(st["gauss13"]), B, P, V, ptr(st["viewmats"]), ptr(st["projmats"]), ptr(st["bg"]), H, W,
            st["scale_modifier"], ptr(st["radii"]), ptr(t["gc"]), ptr(t["ga"]), ptr(st["ws"]), st["L"].total_bytes,
            st["max_instances"], 32, ptr(scratch), scratch.numel(), ptr(grad), stream(dev)), "ga_raster_backward_ex")
        torch.cuda.synchronize()
        return grad

    nbytes = lib.ga_raster_backward_scratch_bytes(B, P, V)
    assert nbytes >= B * V * P * 18 * 4
    clean = run(torch.zeros(nbytes, dtype=torch.uint8, device=dev))
    dirty = torch.full((nbytes + (1 << 20),), 0x7f, dtype=torch.uint8, device=dev)        # 0x7f7f7f7f: a huge float
    dirty[: nbytes // 2].random_(0, 256)
    before = dirty.clone()
    got = run(dirty)
    # the order of the atomics differs from run to run; the rows sum the same partials, so allow rounding
    assert rel_l2(got.cpu().numpy(), clean.cpu().numpy()) <= 1e-6
    used = B * P * 16 * 4
    assert torch.isfinite(dirty[:used].view(torch.float32)).all()        # zeroed before the sums
    assert torch.equal(dirty[used:], before[used:])
