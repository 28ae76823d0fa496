"""The forward's per-instance contribution counts (inst_cnt), which size each instance's records in the backward."""
import numpy as np
import pytest
import torch

from tests.helpers import cameras, scene

pytestmark = pytest.mark.gpu


def test_forward_inst_cnt_sums_match_pixel_lists():
    """With list_k = 32, for every tile whose lists did not overflow, the counts of the tile's instances sum to the
    contributions recorded over its pixels.  Only positions below the tile's deepest contributor are summed: the
    forward stops staging surfels once every pixel is saturated, and the backward reads no count beyond that."""
    from gaussiananything_b200 import raster
    P, H, W, V = 5000, 128, 112, 2
    g = scene(P, 80, 5.0)
    vs, ps, _, _ = cameras(V, start=4)
    dev = torch.device("cuda:0")
    g13 = torch.tensor(g, device=dev)[None]
    vm, pm = torch.tensor(vs, device=dev)[None], torch.tensor(ps, device=dev)[None]
    _, _, _, st = raster.forward_raw(g13, vm, pm, torch.tensor([1.0, 0.5, 0.2], device=dev), H, W, list_k=32)
    L, ws = st["L"], st["ws"]
    gx, gy = (W + 15) // 16, (H + 15) // 16
    T = gx * gy
    wsv = raster.workspace_views(ws, L, 1, P, V, H, W, st["max_instances"], list_k=32)
    tile_start = wsv["tile_start"].cpu().numpy().astype(np.int64)
    last = wsv["n_contrib"][:, 0].cpu().numpy()                                   # [V, H, W]
    flags = wsv["tile_flag"].cpu().numpy()
    n_list = wsv["n_list"].cpu().numpy()
    inst_cnt = wsv["inst_cnt"].cpu().numpy()
    checked = 0
    for v in range(V):
        for ty in range(gy):
            for tx in range(gx):
                t = v * T + ty * gx + tx
                if flags[t]:
                    continue
                ys, xs = slice(ty * 16, ty * 16 + 16), slice(tx * 16, tx * 16 + 16)
                depth = int(last[v, ys, xs].max())
                assert depth <= tile_start[t + 1] - tile_start[t]
                want = int(n_list[v, ys, xs].sum())
                got = int(inst_cnt[tile_start[t]:tile_start[t] + depth].astype(np.int64).sum())
                assert got == want, (v, ty, tx, got, want)
                checked += want > 0
    assert checked > 0
