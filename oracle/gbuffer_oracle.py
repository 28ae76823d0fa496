"""CPU restatement of the G-buffer chunk front end and of the reconstruction metrics (the checker of
gaussiananything_b200/gbuffer.py and csrc/gbuffer_ops.cu; never imported by the product).

`pack` restates the reference's PostProcess._post_process_sample_batch (datasets/g_buffer_objaverse.py:481-702) at
the deployed configuration: reso == reso_encoder == the files' size, ImageNet Normalize, read_normal, Pluecker rays
of the cameras as stored (frame_0_as_canonical=False), append_xyz.  Channels 0-5 are always the fp32 formula (they
are a few roundings of 8-bit values, and the kernel is held to them bit for bit); the rays and the unprojection run
in `dtype`: float64 is the yardstick for the kernel's rounding, float32 repeats the reference's torch operations one
for one and reproduces its output, including the set of xyz values the clip rule zeroes.

A chunk is the dict gaussiananything_b200.gbuffer.read_chunk returns: raw_img, normal uint8 [h, n * w, 3] and alpha
uint8 [h, n * w] with the n views side by side, depth fp32 [n, h, w], c fp32 [n, 25].
"""
import numpy as np
import torch

MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)
XYZ_CLIP = float(np.float32(0.45))          # the fp32 value the reference's clip and comparison use
PSNR_CAP = 100.0


def detile(a, n):
    """[h, n * w, ...] -> [n, h, w, ...]"""
    h = a.shape[0]
    return np.ascontiguousarray(np.moveaxis(a.reshape(h, n, -1, *a.shape[2:]), 1, 0))


def pluecker(c, size, dtype=torch.float64):
    """[6, size, size]: cross(o, d), d with gen_rays' directions (normalise in the camera frame, then rotate)."""
    c2w = torch.from_numpy(np.asarray(c[:16], np.float32).reshape(4, 4)).to(dtype)
    fx, cx, fy, cy = (float(c[i]) for i in (16, 18, 20, 21))
    yy, xx = torch.meshgrid(torch.arange(size, dtype=dtype) + 0.5, torch.arange(size, dtype=dtype) + 0.5, indexing="ij")
    xx = (xx / size - cx) / fx
    yy = (yy / size - cy) / fy
    d = torch.stack((xx, yy, torch.ones_like(xx)), dim=-1)
    d = d / torch.norm(d, dim=-1, keepdim=True)
    d = (c2w[None, :3, :3] @ d.reshape(-1, 3, 1))[..., 0].view(size, size, 3)
    o = c2w[:3, 3].expand(size, size, 3)
    return torch.cat([torch.cross(o, d, dim=-1), d], dim=-1).permute(2, 0, 1)


def sampler_rays(c, size, dtype=torch.float64):
    """RaySampler.forward (nsr/volumetric_rendering/ray_sampler.py:211-271): origins [n, 3], directions [n, size^2, 3].
    The pixel is lifted with the skew term, transformed as a point by the whole c2w, and the origin is subtracted."""
    c = torch.from_numpy(np.asarray(c, np.float32)).to(dtype)
    n = c.shape[0]
    c2w, K = c[:, :16].reshape(n, 4, 4), c[:, 16:25].reshape(n, 3, 3)
    fx, fy, cx, cy, sk = (K[:, 0, 0, None], K[:, 1, 1, None], K[:, 0, 2, None], K[:, 1, 2, None], K[:, 0, 1, None])
    g = torch.arange(size, dtype=dtype) * (1.0 / size) + (0.5 / size)
    vv, uu = torch.meshgrid(g, g, indexing="ij")
    u, v = uu.reshape(1, -1).repeat(n, 1), vv.reshape(1, -1).repeat(n, 1)
    one = torch.ones_like(u)
    lx = (u - cx + cy * sk / fy - sk * v / fy) / fx * one
    ly = (v - cy) / fy * one
    pts = torch.stack((lx, ly, one, one), dim=-1)
    world = torch.bmm(c2w, pts.permute(0, 2, 1)).permute(0, 2, 1)[:, :, :3]
    o = c2w[:, :3, 3]
    return o, torch.nn.functional.normalize(world - o[:, None, :], dim=2)


def unproject(c, depth, dtype=torch.float64):
    """_unproj_depth_given_c (:457-479): o + depth * d, clipped to +-0.45, then 0 where |xyz| == 0.45.  The depth is
    used as stored: a background pixel (0) lands on the camera origin."""
    n, size = depth.shape[0], depth.shape[-1]
    o, d = sampler_rays(c, size, dtype)
    z = torch.from_numpy(np.asarray(depth, np.float32)).to(dtype).reshape(n, -1, 1)
    xyz = (o[:, None, :] + z * d).reshape(n, size, size, 3).permute(0, 3, 1, 2)
    xyz = xyz.clip(-XYZ_CLIP, XYZ_CLIP)
    return torch.where(xyz.abs() == XYZ_CLIP, torch.zeros_like(xyz), xyz)


def pack(chunk, views=None, dtype=torch.float64):
    """dict: img_to_encoder [V, 15, H, W], img [V, 3, H, W] in [-1, 1], alpha, depth, mask [V, 1, H, W], c [V, 25]."""
    n = chunk["c"].shape[0]
    views = list(range(n)) if views is None else [int(v) for v in views]
    c = np.asarray(chunk["c"], np.float32)[views]
    raw = torch.from_numpy(detile(chunk["raw_img"], n)[views]).permute(0, 3, 1, 2) / 255.0          # fp32
    mean, std = torch.tensor(MEAN).view(1, 3, 1, 1), torch.tensor(STD).view(1, 3, 1, 1)
    rgb = (raw - mean) / std
    nm = detile(chunk["normal"], n)[views].astype(np.float32) / 255.0
    nm = nm * 2 - 1
    nm = np.stack([-nm[..., 0], -nm[..., 2], nm[..., 1]], axis=-1)                                  # unity2blender_fix
    nm = torch.from_numpy(nm).permute(0, 3, 1, 2)
    depth = np.asarray(chunk["depth"], np.float32)[views]
    size = depth.shape[-1]
    rays = torch.stack([pluecker(ci, size, dtype) for ci in c], 0)
    xyz = unproject(c, depth, dtype)
    enc = torch.cat([rgb.to(dtype), nm.to(dtype), rays, xyz], 1)
    d = torch.from_numpy(depth)[:, None]
    alpha = torch.from_numpy(detile(chunk["alpha"], n)[views] / 255.0).float()[:, None]
    return {"img_to_encoder": enc, "img": raw * 2 - 1, "alpha": alpha, "depth": d, "mask": (d > 0).float(),
            "c": torch.from_numpy(c)}


def metric_table(render, targets):
    """fp64 [V, 8] of the sums include/ga_b200.h states for ga_recon_metrics.  render: image, rend_normal [V, 3, H, W],
    depth, alpha [V, 1, H, W]; targets: img, normal [V, 3, H, W], depth, alpha, mask [V, 1, H, W]."""
    r = {k: render[k].detach().double().cpu() for k in ("image", "depth", "alpha", "rend_normal")}
    t = {k: targets[k].detach().double().cpu() for k in ("img", "depth", "alpha", "mask", "normal")}
    s = lambda x: x.flatten(1).sum(1)
    pi, gi = r["alpha"] > 0.5, t["alpha"] > 0.5
    dot = (r["rend_normal"] * t["normal"]).sum(1, keepdim=True)
    cols = [s((r["image"] - (t["img"] + 1) * 0.5) ** 2), s(t["mask"] * (r["depth"] - t["depth"]).abs()), s(t["mask"]),
            s(t["mask"] * (1 - dot)), s((r["alpha"] - t["alpha"]).abs()), s((pi & gi).double()), s((pi | gi).double()),
            s(torch.ones_like(t["mask"]))]
    return torch.stack(cols, 1)


def derive(table):
    """Per-view numbers from the table: PSNR on [0, 1] (PSNR_CAP dB where the error is exactly zero), mean depth L1
    and normal error over the foreground (0 where the view has no foreground), mean alpha L1, alpha IoU at 0.5
    (1 where neither map has a pixel above 0.5)."""
    t = table.double()
    mse = t[:, 0] / (3 * t[:, 7])
    fg = t[:, 2].clamp_min(1)
    return {"psnr": torch.where(mse > 0, (-10 * torch.log10(mse.clamp_min(1e-300))).clamp_max(PSNR_CAP),
                                torch.full_like(mse, PSNR_CAP)),
            "depth_l1": torch.where(t[:, 2] > 0, t[:, 1] / fg, torch.zeros_like(mse)),
            "normal_error": torch.where(t[:, 2] > 0, t[:, 3] / fg, torch.zeros_like(mse)),
            "alpha_l1": t[:, 4] / t[:, 7],
            "iou": torch.where(t[:, 6] > 0, t[:, 5] / t[:, 6].clamp_min(1), torch.ones_like(mse)),
            "fg_pixels": t[:, 2]}
