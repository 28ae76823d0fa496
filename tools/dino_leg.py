"""Time the DINOv2 image conditioner (SURVEY.md 8f row N3) on the GPU and one image -> 3D sample through it:

    python tools/dino_leg.py

Prints one JSON line: the card and its power limit (read in the same run); the encoder's ms per image at batch 1
and 4 (CUDA-graph replay, warmed up, >= 2 s of timed work per batch size, device events) and TFLOP/s from
dino.encode_flops; the unfused PyTorch stand-in (baseline/gpu_standin.py TorchDino: bf16 autocast nn.Linear +
F.scaled_dot_product_attention) at the same batch sizes; and the cascade per sample from an image -- conditioner,
DiT-L stage 1 and stage 2 (2 x 249 Euler NFE, CFG 4), VAE decode, 8 views of 512^2 -- beside the same cascade fed
synthetic context tokens (no conditioner), both measured in this run.  Random weights (no checkpoint is read).
The input image is a 518^2 rendering of a surfel scene by the library's rasteriser.
Needs a CUDA device; fails without one.
"""
import json
import math
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MIN_SECONDS = 2.0


def card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        watts = float(r.stdout.strip().splitlines()[0])
    except Exception:
        watts = None
    return name, watts


def time_replay(fn, min_seconds=MIN_SECONDS):
    """(ms per call, reps): device events around >= min_seconds of back-to-back calls, after a warm-up."""
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    reps = max(10, math.ceil(min_seconds / max(e0.elapsed_time(e1) * 1e-3, 1e-6)))
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps, reps


def rendered_image(dev, size=518):
    """A [1, 3, size, size] image in [-1, 1]: one view of a random surfel scene rendered by the library."""
    from gaussiananything_b200 import raster
    from tests.helpers import cameras, scene
    g13 = torch.tensor(scene(20000, 3, 6.0), device=dev)[None]
    vs, ps, _, _ = cameras(1)
    color, _, _ = raster.rasterize_surfels_batched(g13, torch.tensor(vs, device=dev)[None], torch.tensor(ps, device=dev)[None],
                                                   torch.ones(3, device=dev), size, size, 1.0)
    return (color[0, :1].clamp(0, 1) * 2 - 1).contiguous()


def encoder_leg(dev, enc, sd):
    from baseline import gpu_standin as gs
    from gaussiananything_b200 import dino
    out = {}
    for B in (1, 4):
        img = torch.rand(B, 3, 518, 518, device=dev) * 2 - 1
        enc.encode(img)                                            # captures the graph for (B, 518, 518)
        g = enc._graphs[(B, 518, 518)][0]
        ms, reps = time_replay(g.replay)
        out["B%d" % B] = {"ms_per_batch": ms, "ms_per_image": ms / B, "reps": reps,
                          "tflops": dino.encode_flops(B, enc.depth) / (ms * 1e-3) / 1e12}
        out["standin_B%d" % B] = gs.time_torch_dino(dev, sd, B, MIN_SECONDS)
    return out


def cascade_leg(dev, enc, img, samples=2):
    """Seconds per sample of the whole cascade, with the conditioner on `img` and with synthetic context tokens."""
    from gaussiananything_b200 import dino, dit, transport as tr
    from gaussiananything_b200.gs_surfel import GaussianRenderer2DGS
    from gaussiananything_b200.vae_decoder import SurfelDecoder, random_state_dict
    from tests.helpers import cameras
    torch.manual_seed(0)
    N, V, RES = 768, 8, 512
    emb = dino.FrozenDinov2ImageEmbedder(arch="vitl", inp_size=518, output_cls=True, encoder=enc)
    emb.input_key = "img"
    cond1 = dino.GeneralConditioner([emb])
    cond2 = dino.GeneralConditioner([emb, {"input_key": "fps-xyz", "ucg_rate": 0.0,
                                           "target": "sgm.modules.encoders.modules.PCD_Scaler",
                                           "params": {"scaling_factor": 0.45}}])
    mk = lambda name, cin: dit.DiT_models[name](input_size=32, num_classes=0, learn_sigma=False, in_channels=cin,
                                                context_dim=1024, roll_out=True, pooling_ctx_dim=768).randomize_zero_init_().to(dev).eval()
    m1, m2 = mk("DiT-PixArt-PCD-CLAY-L", 3), mk("DiT-PixArt-PCD-CLAY-stage2-L", 10)
    fn = tr.Sampler(tr.create_transport("GVP", "velocity", None, None, None, "lognorm")).sample_ode(
        sampling_method="euler", num_steps=250)
    dec = SurfelDecoder(random_state_dict(768, 12, 10, seed=0), 12, 12, device=dev)
    rnd = GaussianRenderer2DGS(RES, 3, {})
    vs, ps, cs, tf = cameras(V)
    cv, cp = torch.tensor(vs, device=dev)[None], torch.tensor(ps, device=dev)[None]
    pos = torch.tensor(cs, device=dev)[None]
    syn_c, syn_v = torch.randn(1, 1369, 1024, device=dev), torch.randn(1, 1024, device=dev)
    cfg = lambda c, uc: {k: torch.cat([c[k], uc[k]], 0) for k in c}

    def one_sample(with_conditioner):
        if with_conditioner:
            c, uc = cond1.get_unconditional_conditioning({"img": img}, force_uc_zero_embeddings=["img"])
        else:
            c = {"img_crossattn": syn_c, "img_vector": syn_v}
            uc = {k: torch.zeros_like(v) for k, v in c.items()}
        z = torch.randn(1, N, 3, device=dev)
        pts = fn(torch.cat([z, z], 0), m1.forward_with_cfg, context=cfg(c, uc), cfg_scale=4.0)[-1][:1]
        pts = (pts * 0.164).clamp(-0.45, 0.45)                     # stage-1 un-normalisation
        if with_conditioner:
            c, uc = cond2.get_unconditional_conditioning({"img": img, "fps-xyz": pts}, force_uc_zero_embeddings=["img-xyz"])
        else:
            c = dict(c, **{"fps-xyz": pts / 0.45})
            uc = c
        z2 = torch.randn(1, N, 10, device=dev)
        lat = fn(torch.cat([z2, z2], 0), m2.forward_with_cfg, context=cfg(c, uc), cfg_scale=4.0)[-1][:1]
        surf = dec.decode(lat, pts)["gaussians_upsampled_3"]
        return rnd.render(surf, cv, cp, pos, tf)

    res = {}
    with torch.no_grad():
        for tag, wc in (("with_conditioner", True), ("synthetic_context_no_conditioner", False)):
            one_sample(wc)                                          # warm-up: weight packs, K/V, graphs
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            for _ in range(samples):
                o = one_sample(wc)
            o["image"][:, :1, :, :8, :8].cpu()
            torch.cuda.synchronize(dev)
            dt = (time.perf_counter() - t0) / samples
            assert torch.isfinite(o["image"]).all()
            res[tag] = {"seconds_per_sample": dt, "samples_per_s": 1.0 / dt}
    # the conditioner's share alone: stage-1 and stage-2 get_unconditional_conditioning on one image
    res["conditioner_ms_per_sample"] = 2 * time_replay(lambda: cond1.get_unconditional_conditioning(
        {"img": img}, force_uc_zero_embeddings=["img"]), 0.5)[0]
    res["config"] = ("image 518^2 -> DINOv2 conditioner (stage 1 c / zero uc, stage 2 uc == c) -> DiT-PixArt-PCD-CLAY-L "
                     "+ ...-stage2-L (L24 D1024 H16), N=768, M=1369, 250-point Euler grids (2 x 249 NFE), CFG 4.0, bf16 -> "
                     "VAE decode (73 728 surfels) -> %d views of %d^2; one sample at a time, one GPU, random weights" % (V, RES))
    del m1, m2, dec
    torch.cuda.empty_cache()
    return res


def main():
    if not torch.cuda.is_available():
        raise SystemExit("tools/dino_leg.py needs a CUDA device")
    from gaussiananything_b200 import dino
    dev = torch.device("cuda:0")
    name, watts = card()
    sd = dino.random_state_dict(24, seed=0)
    enc = dino.Dinov2Encoder(sd, dev)
    out = {"what": "DINOv2 ViT-L/14-reg4 image conditioner (518^2, 1374 tokens, 24 blocks) on libga_b200.so",
           "gpu": name, "power_limit_w": watts, "flop_per_image": dino.encode_flops(1, 24)}
    out["encoder"] = encoder_leg(dev, enc, sd)
    img = rendered_image(dev)
    out["cascade"] = cascade_leg(dev, enc, img)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
