"""Host restatements for the surface point clouds (include/ga_b200.h Part 10): the chunk keep rule of
save_pcd_from_depth on oracle/gbuffer_oracle.unproject, and pytorch3d's padded farthest-point sampling on
oracle/vae_encoder_oracle.fps.  Test code only; the product never imports it."""
import numpy as np
import torch

from oracle import gbuffer_oracle as go
from oracle import vae_encoder_oracle as vo


def surface_points(chunk, views=None, alpha_min=255, min_depth=1.05, dtype=torch.float64):
    """[N, 3] in `dtype`: the unprojected xyz (clipped, 0 on the clip value) of the pixels with alpha >= alpha_min,
    depth >= min_depth and all three coordinates nonzero, in view order, then row-major pixel order."""
    n = chunk["c"].shape[0]
    views = list(range(n)) if views is None else [int(v) for v in views]
    c = np.asarray(chunk["c"], np.float32)[views]
    depth = np.asarray(chunk["depth"], np.float32)[views]
    xyz = go.unproject(c, depth, dtype).permute(0, 2, 3, 1)                     # [V, H, W, 3]
    alpha = torch.from_numpy(go.detile(np.asarray(chunk["alpha"]), n)[views])
    keep = (alpha >= alpha_min) & (torch.from_numpy(depth) >= min_depth) & (xyz != 0).all(-1)
    return xyz[keep]


def fps_padded(pcd, lengths, K, start):
    """pcd [B, N, 3], lengths [B], start [B] -> (xyz [B, K, 3], idx [B, K] int64): cloud b is pcd[b, :lengths[b]];
    past min(K, lengths[b]) the entries are -1 and 0, as pytorch3d pads."""
    B = pcd.shape[0]
    idx = torch.full((B, K), -1, dtype=torch.int64)
    xyz = torch.zeros(B, K, 3)
    for b in range(B):
        n = int(lengths[b])
        k = min(K, n)
        if k:
            x, i = vo.fps(pcd[b:b + 1, :n], k, start[b:b + 1])
            xyz[b, :k], idx[b, :k] = x[0], i[0]
    return xyz, idx
