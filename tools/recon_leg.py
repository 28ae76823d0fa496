"""Time the G-buffer chunk front end and the VAE reconstruction round trip on the GPU, on the committed chunk
(tests/golden/gbuffer_chunk):

    python tools/recon_leg.py

Prints one JSON line: the card and its power limit (read in the same run); ga_gbuffer_pack for the 8 encoder views,
with and without the render targets, as the bare launch into buffers allocated once and as the gbuffer.pack call, and
for all 16 views, from device-resident inputs (microseconds per call and the bytes it must move over that time); the
same encoder input built by the sequence of eager torch operations the kernel replaces (`torch_pack` below, checked
against the kernel in the same run); ga_recon_metrics for 8 views; and the whole 'reconstruct_chunk' call (read the
files, pack, encode, decode to 73 728 surfels, render 16 views at 512^2, metrics).  The packers alternate inside one
process; every timing is device events around >= 1 s of back-to-back calls after a warm-up.  Random weights (no
checkpoint is read), so the reconstruction metrics it prints say nothing
about quality.  Needs a CUDA device.
"""
import ctypes as C
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.dino_leg import card, time_replay  # noqa: E402

CHUNK = os.path.join(ROOT, "tests", "golden", "gbuffer_chunk")
H = 512


def torch_pack(d, views):
    """img_to_encoder [V, 15, H, W] with eager torch operations on the device, in the reference's order of steps."""
    n = d["c"].shape[0]
    vi = torch.as_tensor(views, device=d["c"].device)
    c = d["c"][vi]
    V = len(views)
    detile = lambda a: a.reshape(H, n, H, -1).permute(1, 3, 0, 2)[vi]
    rgb = detile(d["raw_img"]) / 255.0
    mean = torch.tensor([0.485, 0.456, 0.406], device=c.device).view(1, 3, 1, 1)
    std = torch.tensor([0.229, 0.224, 0.225], device=c.device).view(1, 3, 1, 1)
    rgb = (rgb - mean) / std
    nm = (detile(d["normal"]) / 255.0) * 2 - 1
    nm = torch.stack([-nm[:, 0], -nm[:, 2], nm[:, 1]], 1)
    c2w, K = c[:, :16].reshape(V, 4, 4), c[:, 16:].reshape(V, 3, 3)
    fx, fy, cx, cy, sk = (K[:, 0, 0, None], K[:, 1, 1, None], K[:, 0, 2, None], K[:, 1, 2, None], K[:, 0, 1, None])
    g = (torch.arange(H, device=c.device, dtype=torch.float32) + 0.5) / H
    vv, uu = torch.meshgrid(g, g, indexing="ij")
    u, v = uu.reshape(1, -1), vv.reshape(1, -1)
    dirs = torch.stack(((u - cx) / fx, (v - cy) / fy, torch.ones(V, H * H, device=c.device)), -1)
    dirs = dirs / torch.norm(dirs, dim=-1, keepdim=True)
    dirs = torch.bmm(dirs, c2w[:, :3, :3].transpose(1, 2))
    o = c2w[:, None, :3, 3].expand(V, H * H, 3)
    rays = torch.cat([torch.cross(o, dirs, dim=-1), dirs], -1).reshape(V, H, H, 6).permute(0, 3, 1, 2)
    one = torch.ones(V, H * H, device=c.device)
    lx = (u - cx + cy * sk / fy - sk * v / fy) / fx * one
    ly = (v - cy) / fy * one
    pts = torch.stack((lx, ly, one, one), -1)
    world = torch.bmm(c2w, pts.permute(0, 2, 1)).permute(0, 2, 1)[:, :, :3]
    r = torch.nn.functional.normalize(world - o, dim=2)
    xyz = (o + d["depth"][vi].reshape(V, -1, 1) * r).reshape(V, H, H, 3).permute(0, 3, 1, 2).clip(-0.45, 0.45)
    xyz = torch.where(xyz.abs() == 0.45, 0, xyz)
    return torch.cat([rgb, nm, rays, xyz], 1)


def pack_bytes(V, targets):
    """Bytes one ga_gbuffer_pack launch has to read and write for V views of 512^2."""
    px = V * H * H
    return px * (15 * 4 + 3 + 3 + 4) + (px * (6 * 4 + 1) if targets else 0)


def main():
    assert torch.cuda.is_available(), "recon_leg.py measures on the GPU"
    from gaussiananything_b200 import _lib, gbuffer, vae_decoder as vd, vae_encoder as ve
    name, watts = card()
    dev = torch.device("cuda:0")
    chunk = gbuffer.read_chunk(CHUNK)
    d = gbuffer.to_device(chunk, dev)
    res = {"card": name, "power_limit_w": watts}

    views8, views16 = list(range(8)), list(range(16))
    enc_k, _, _ = gbuffer.pack(d, views8, dev)
    enc_t = torch_pack(d, views8)
    diff = (enc_k - enc_t).abs()
    res["kernel_vs_torch"] = {"max_abs_rgb_normal": float(diff[:, :6].max()), "max_abs_rays": float(diff[:, 6:12].max()),
                              "xyz_zero_set_differs_at": int(((enc_k[:, 12:] == 0) != (enc_t[:, 12:] == 0)).sum())}
    del enc_k, enc_t, diff
    # the two packers in turn, twice, so that a drift of the clocks shows as a spread.  "launch_*" is the kernel alone
    # into buffers allocated once; the other kernel rows are gbuffer.pack, which also allocates its outputs and
    # uploads the view list
    p = lambda x: C.c_void_p(x.data_ptr())
    vi = torch.tensor(views8, dtype=torch.int32, device=dev)
    enc_b = torch.empty(8, 15, H, H, device=dev)
    tb = [torch.empty(8, ch, H, H, device=dev) for ch in (3, 1, 1, 1)]
    st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    launch = lambda *t: _lib.check(_lib.lib().ga_gbuffer_pack(
        p(d["raw_img"]), p(d["normal"]), p(d["alpha"]), p(d["depth"]), p(d["c"]), 16, H, H, p(vi), 8, p(enc_b),
        *(t or [None] * 4), st), "ga_gbuffer_pack")
    runs = {"launch_8_views": lambda: launch(),
            "launch_8_views_with_targets": lambda: launch(*[p(x) for x in tb]),
            "kernel_8_views_with_targets": lambda: gbuffer.pack(d, views8, dev),
            "torch_8_views": lambda: torch_pack(d, views8),
            "kernel_8_views": lambda: gbuffer.pack(d, views8, dev, with_targets=False),
            "kernel_16_views_with_targets": lambda: gbuffer.pack(d, views16, dev)}
    us = {k: [] for k in runs}
    for _ in range(2):
        for k, fn in runs.items():
            ms, _ = time_replay(fn, min_seconds=1.0)
            us[k].append(round(ms * 1e3, 1))
    nbytes = {"launch_8_views": pack_bytes(8, False), "launch_8_views_with_targets": pack_bytes(8, True),
              "kernel_8_views_with_targets": pack_bytes(8, True), "kernel_8_views": pack_bytes(8, False),
              "kernel_16_views_with_targets": pack_bytes(16, True)}
    res["pack_us_per_call"] = us
    res["pack_gb_per_s"] = {k: round(b / (min(us[k]) * 1e-6) / 1e9, 1) for k, b in nbytes.items()}
    res["pack_speedup_vs_torch"] = round(min(us["torch_8_views"]) / min(us["kernel_8_views"]), 1)

    _, t, _ = gbuffer.pack(d, list(range(8, 16)), dev)
    g = torch.Generator(device=dev).manual_seed(0)
    near = lambda x: x + 0.1 * (torch.rand(x.shape, generator=g, device=dev) - 0.5)
    r = {"image": near((t["img"] + 1) / 2), "depth": near(t["depth"]), "alpha": near(t["alpha"]),
         "rend_normal": near(t["normal"])}
    ms, _ = time_replay(lambda: gbuffer.metric_table(r, t), min_seconds=1.0)
    res["metrics_8_views_us"] = round(ms * 1e3, 1)
    res["metrics_gb_per_s"] = round(8 * H * H * 18 * 4 / (ms * 1e-3) / 1e9, 1)

    enc = ve.SurfelEncoder(ve.random_state_dict(seed=0), num_frames=8, latent_num=768)
    dec = vd.SurfelDecoder(vd.random_state_dict(D=768, depth=12), num_heads=12, depth=12)
    ae = vd.SurfelAE(dec, encoder=enc)
    ply = os.path.join(CHUNK, "fps-4096.ply")
    call = lambda src: ae(behaviour="reconstruct_chunk", chunk=src, pcd=ply, fps_start=torch.tensor([0]),
                          generator=torch.Generator().manual_seed(0))
    ms_files, _ = time_replay(lambda: call(CHUNK), min_seconds=2.0)
    ms_decoded, _ = time_replay(lambda: call(chunk), min_seconds=2.0)
    out = call(chunk)
    res["reconstruct_chunk_ms"] = {"from_files": round(ms_files, 1), "from_decoded_chunk": round(ms_decoded, 1)}
    res["random_weight_metrics_eval_views"] = {k: [round(float(x), 3) for x in v]
                                               for k, v in out["eval"]["metrics"].items() if k != "fg_pixels"}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
