"""Surface point clouds on the GPU: the clouds the reference's scripts/save_pcd.py and save_pcd_from_gs.py make with
pytorch3d, on the library's kernels (include/ga_b200.h Part 10).

  sample_farthest_points   pytorch3d.ops.sample_farthest_points: ga_fps_ex (one CTA per cloud where a cloud fits
                           one, else a cooperative grid per call), clouds of up to 4M points and K up to 32 768
  chunk_surface_points     a G-buffer chunk's depth maps fused into one cloud (ga_chunk_surface_points): the
                           encoder's xyz channels of the kept pixels, in view-major, row-major order
  chunk_surface_pcd        fuse, then farthest-point sample K points from index 0: save_pcd_from_depth's fps-K.ply
  gaussians_pcd            decoded surfels with opacity >= min_opacity, sampled likewise: save_pcd_from_gs's fps-K.ply
  write_ply                binary little-endian x, y, z floats (gbuffer.read_fps_pcd reads them back)
"""
import os

import numpy as np
import torch

from . import _lib
from ._launch import ptr, stream
from .gbuffer import read_chunk, to_device

ALPHA_MIN = 255          # save_pcd_from_depth's alpha_mask == 1 on the 8-bit alpha.jpg
MIN_DEPTH = 1.05         # its depth < 1.05 outlier filter


def _cuda(t, what):
    if not isinstance(t, torch.Tensor) or t.device.type != "cuda":
        raise RuntimeError("%s runs on a CUDA device (there is no CPU fallback)" % what)


def sample_farthest_points(points, lengths=None, K=50, random_start_point=False, generator=None):
    """pytorch3d.ops.sample_farthest_points on the GPU.  points [B, N, 3]; lengths [B] (points of each cloud, None: N);
    K an int or one per cloud; random_start_point: start cloud b at torch.randint(lengths[b], generator=generator)
    instead of index 0.  Returns (xyz [B, max K, 3] in points' dtype, idx [B, max K] int64); the entries past
    min(K_b, lengths[b]) are -1 and 0, as pytorch3d pads.  Distances are fp32, (dx*dx + dy*dy) + dz*dz with ties to the
    lowest index (ga_fps_ex)."""
    _cuda(points, "pcd.sample_farthest_points")
    if points.dim() != 3 or points.shape[2] != 3:
        raise ValueError("points must be [B, N, 3], got %s" % (tuple(points.shape),))
    B, N, _ = points.shape
    lens = (torch.full((B,), N, dtype=torch.int64) if lengths is None
            else torch.as_tensor(lengths).to("cpu", torch.int64).reshape(-1))
    if lens.shape != (B,):
        raise ValueError("lengths must be [%d], got %s" % (B, tuple(lens.shape)))
    if int(lens.min()) < 0 or int(lens.max()) > N:
        raise ValueError("lengths must lie in [0, %d]" % N)
    Ks = torch.as_tensor(K).to("cpu", torch.int64).reshape(-1) if not isinstance(K, int) else torch.full((B,), K)
    if Ks.shape != (B,) and Ks.numel() != 1:
        raise ValueError("K must be an int or one value per cloud")
    Ks = Ks.expand(B)
    if int(Ks.min()) <= 0:
        raise ValueError("K must be positive")
    Kmax = int(Ks.max())
    start = torch.zeros(B, dtype=torch.int32)
    if random_start_point:
        for b in range(B):
            start[b] = int(torch.randint(high=max(int(lens[b]), 1), size=(1,), generator=generator))
    dev = points.device
    pts = points.to(torch.float32).contiguous()
    idx = torch.empty(B, Kmax, dtype=torch.int32, device=dev)
    xyz = torch.empty(B, Kmax, 3, device=dev)
    L = _lib.lib()
    ws = torch.empty(L.ga_fps_ex_workspace_bytes(B, N, Kmax), dtype=torch.uint8, device=dev)
    ld = None if lengths is None else lens.to(dev, torch.int32)
    with torch.cuda.device(dev):
        _lib.check(L.ga_fps_ex(ptr(pts), ptr(ld), B, N, Kmax, ptr(start.to(dev)), ptr(idx), ptr(xyz), ptr(ws), ws.numel(),
                               stream(dev)), "ga_fps_ex")
    if int(Ks.min()) < Kmax:                                   # per-cloud K: FPS is prefix-stable, so cut and pad
        cut = torch.arange(Kmax)[None] >= Ks[:, None]
        cut = cut.to(dev)
        idx = idx.masked_fill(cut, -1)
        xyz = xyz.masked_fill(cut[..., None], 0.0)
    return xyz.to(points.dtype), idx.long()


def chunk_surface_points(chunk, views=None, alpha_min=ALPHA_MIN, min_depth=MIN_DEPTH, device="cuda"):
    """The chunk's surface points, fp32 [N, 3] on the device: every pixel of `views` (default: all) with alpha >=
    alpha_min (uint8), depth >= min_depth and all three unprojected coordinates nonzero, unprojected exactly as
    gbuffer.pack's xyz channels 12-14 (clipped to +-0.45, so a kept coordinate is strictly inside), in view order,
    then row-major pixel order.  chunk: a folder or read_chunk's dict (host arrays or to_device's tensors)."""
    if isinstance(chunk, (str, os.PathLike)):
        chunk = read_chunk(chunk)
    dev = torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError("pcd.chunk_surface_points runs on a CUDA device (there is no CPU fallback)")
    n, h, w = chunk["depth"].shape
    views = list(range(n)) if views is None else [int(v) for v in views]
    if not views or min(views) < 0 or max(views) >= n:
        raise IndexError("pcd.chunk_surface_points: views %r outside the chunk's %d views" % (views, n))
    if not 0 <= int(alpha_min) <= 255:
        raise ValueError("alpha_min is an 8-bit alpha threshold, got %r" % alpha_min)
    d = to_device({k: chunk[k] for k in ("alpha", "depth", "c")}, dev)
    V = len(views)
    vi = torch.tensor(views, dtype=torch.int32, device=dev)
    pts = torch.empty(V * h * w, 3, device=dev)
    count = torch.empty(1, dtype=torch.int32, device=dev)
    L = _lib.lib()
    scratch = torch.empty(L.ga_chunk_surface_points_scratch_bytes(V, h, w), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(L.ga_chunk_surface_points(ptr(d["alpha"]), ptr(d["depth"]), ptr(d["c"]), n, h, w, ptr(vi), V,
                                             int(alpha_min), float(min_depth), ptr(pts), ptr(count), ptr(scratch),
                                             scratch.numel(), stream(dev)), "ga_chunk_surface_points")
    return pts[:int(count)]


def chunk_surface_pcd(chunk, K=4096, views=None, device="cuda", **thresholds):
    """save_pcd_from_depth's fps-K.ply: chunk_surface_points (thresholds: alpha_min, min_depth) sampled to K points
    by farthest-point sampling from index 0.  fp32 [K, 3] on the device (zero rows past the cloud's size, as
    pytorch3d pads)."""
    pts = chunk_surface_points(chunk, views, device=device, **thresholds)
    if pts.shape[0] == 0:
        raise ValueError("pcd.chunk_surface_pcd: no pixel of the chunk passes the keep rule")
    return sample_farthest_points(pts[None], K=K)[0][0]


def gaussians_pcd(gauss13, K=4096, min_opacity=0.005):
    """save_pcd_from_gs's fps-K.ply for each item: the xyz of the surfels whose opacity (column 3, as the rasteriser
    takes it) is not below min_opacity, sampled to K points by farthest-point sampling from index 0.
    gauss13 [B, P, 13] (or [P, 13]) on the device -> fp32 [B, K, 3] (or [K, 3])."""
    _cuda(gauss13, "pcd.gaussians_pcd")
    g = gauss13[None] if gauss13.dim() == 2 else gauss13
    keep = ~(g[..., 3] < min_opacity)                      # the reference drops opacity < min_opacity only
    lengths = keep.sum(1)
    # kept points first, in their order: a stable sort of the drop flags
    order = torch.sort((~keep).to(torch.uint8), dim=1, stable=True)[1]
    xyz = torch.gather(g[..., :3].float(), 1, order[..., None].expand(-1, -1, 3)).contiguous()
    out = sample_farthest_points(xyz, lengths=lengths, K=K)[0]
    return out[0] if gauss13.dim() == 2 else out


def write_ply(path, xyz):
    """Writes xyz [N, 3] as a binary little-endian PLY of float x, y, z vertices (what point-cloud-utils'
    save_mesh_v writes for the reference's fps-K.ply)."""
    a = (xyz.detach().cpu().numpy() if isinstance(xyz, torch.Tensor) else np.asarray(xyz)).astype("<f4")
    if a.ndim != 2 or a.shape[1] != 3:
        raise ValueError("write_ply: xyz must be [N, 3], got %s" % (a.shape,))
    head = ("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\n"
            "property float z\nend_header\n" % a.shape[0]).encode("ascii")
    with open(path, "wb") as f:
        f.write(head + np.ascontiguousarray(a).tobytes())
