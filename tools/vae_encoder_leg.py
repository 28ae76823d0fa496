"""Time the 3D VAE encoder on the GPU and the VAE reconstruction round trip through it:

    python tools/vae_encoder_leg.py

Prints one JSON line: the card and its power limit (read in the same run); the encoder's ms per sample at B = 1 and 2
(8 views of 512^2, 4 096 points, 768 latents; CUDA-graph replay, warmed up, >= 2 s of timed work, device events) and
TFLOP/s from vae_encoder.encode_flops; the per-category split of one encode from torch.profiler (conv / GroupNorm /
multi-view attention block / readout); the unfused bf16 PyTorch stand-in (baseline/gpu_standin.py TorchVaeEncoder) at
the same sizes; and the reconstruction round trip at B = 1: encode -> decode to 73 728 surfels -> 50 orbit views at
512^2 -> TSDF mesh.  Random weights (no checkpoint is read).  Needs a CUDA device.
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.dino_leg import card, time_replay  # noqa: E402

V, H, NP, K = 8, 512, 4096, 768


def inputs(B, seed=0):
    g = torch.Generator().manual_seed(seed)
    img = torch.randn(B * V, 15, H, H, generator=g).cuda()
    pcd = (torch.rand(B, NP, 3, generator=g) - 0.5).cuda()
    return img, pcd, torch.arange(B) * 7


def category(name):
    n = name.lower()
    if "conv3x3" in n:
        return "conv3x3"
    if "gn_" in n:
        return "groupnorm"
    if "attn_fwd" in n or "layernorm" in n or "gemm" in n:
        return "gemm_attention"
    return "other"


def profile_split(enc, img, pcd, start):
    from torch.profiler import ProfilerActivity, profile
    enc.use_graph = False
    enc.encode(img, pcd, start)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        enc.encode(img, pcd, start)
        torch.cuda.synchronize()
    enc.use_graph = True
    split = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t:
            c = category(ev.key)
            split[c] = split.get(c, 0.0) + t / 1e3
    return {k: round(v, 3) for k, v in sorted(split.items())}


def round_trip(enc, img, pcd, start):
    from gaussiananything_b200 import mesh, vae_decoder as vd
    dec = vd.SurfelDecoder(vd.random_state_dict(D=768, depth=12), num_heads=12, depth=12)
    ae = vd.SurfelAE(dec, encoder=enc)
    cams = mesh.uni_mesh_path(10)
    setup = mesh.view_setup(cams, 512, 512)

    def once():
        out = ae(img=img, behaviour="enc_dec_wo_triplane", pcd=pcd, fps_start=start,
                 generator=torch.Generator().manual_seed(0))
        _, r = mesh.render_orbit(out["gaussians_upsampled_3"], cams, 512)
        m, _ = mesh.fuse(r["image"][0], r["depth"][0, :, 0], r["alpha"][0, :, 0], setup)
        return mesh.post_process_mesh(m), out["gaussians_upsampled_3"].shape[1]
    once()
    ts = []
    for _ in range(3):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        post, n_surfels = once()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[1], n_surfels, int(post.triangles.shape[0])


def main():
    assert torch.cuda.is_available(), "vae_encoder_leg.py measures on the GPU"
    from baseline.gpu_standin import TorchVaeEncoder
    from gaussiananything_b200 import vae_encoder as ve
    name, watts = card()
    sd = ve.random_state_dict(seed=0)
    enc = ve.SurfelEncoder(sd, num_frames=V, latent_num=K)
    standin = TorchVaeEncoder(sd, num_frames=V, latent_num=K)
    res = {"card": name, "power_limit_w": watts, "tflop_per_sample": ve.encode_flops(1, V, H, H) / 1e12}
    for B in (1, 2):
        img, pcd, start = inputs(B, B)
        ms, reps = time_replay(lambda: enc.encode(img, pcd, start))
        sms, _ = time_replay(lambda: standin.encode(img, pcd, start), min_seconds=1.0)
        res["B%d" % B] = {"ms_per_sample": round(ms / B, 3), "tflops": round(ve.encode_flops(B, V, H, H) / ms / 1e9, 1),
                          "reps": reps, "standin_ms_per_sample": round(sms / B, 3),
                          "speedup_vs_standin": round(sms / ms, 2)}
        if B == 1:
            res["B1"]["profile_ms"] = profile_split(enc, img, pcd, start)
    img, pcd, start = inputs(1, 1)
    ms, n_surfels, n_tri = round_trip(enc, img, pcd, start)
    res["round_trip"] = {"ms": round(ms, 1), "surfels": n_surfels, "views": 50, "triangles": n_tri}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
