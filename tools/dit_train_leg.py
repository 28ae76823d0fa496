"""One flow-matching training step of the image-to-3D DiT-L (stage 1 and stage 2) on the library's kernels
(gaussiananything_b200/dit_grad.py model_forward, include/ga_b200.h Parts 12-15) against the torch stand-in.

    python tools/dit_train_leg.py [--json out.json] [--steps 10] [--configs stage1-B4,stage2-B8,...]

A step is Transport.training_losses (Linear path, velocity) on the model, backward, clip_grad_norm_(1.0) and AdamW
(lr 1e-4, weight decay 0.05), all under bf16 autocast, as the reference trains.  The stand-in is the oracle model
(oracle/dit_oracle.forward on the same nn.Parameters) under torch bf16 autocast with SDPA, the stand-in the block
profile uses.  Ours and the stand-in alternate twice in one process; step time is device events around `steps` steps
after two warm-up steps.  The card's name and power limit are read in the same call.  Peak memory is the allocator's
high-water mark over one step above what was allocated before it.  A separate profiled step of ours gives the launch
count and each Part 15 kernel's time beside its byte floor at 3.35 TB/s; `-Xptxas -v` of csrc/dit_model_grad.cu
gives the new kernels' registers and spills.
"""
import argparse
import functools
import json
import os
import re
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gaussiananything_b200 import dit, dit_grad  # noqa: E402
from gaussiananything_b200.transport import create_transport  # noqa: E402
from oracle import dit_oracle  # noqa: E402

N, M, HBM = 768, 1369, 3.35e12
CONFIGS = {"stage1-B4": ("DiT-PixArt-PCD-CLAY-L", 4), "stage1-B8": ("DiT-PixArt-PCD-CLAY-L", 8),
           "stage2-B4": ("DiT-PixArt-PCD-CLAY-stage2-L", 4), "stage2-B8": ("DiT-PixArt-PCD-CLAY-stage2-L", 8)}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        watts = float(r.stdout.strip().splitlines()[0])
    except Exception:
        watts = None
    return name, watts


def build(arch, B, dev):
    torch.manual_seed(0)
    m = dit.DiT_models[arch](input_size=32, num_classes=0, learn_sigma=False, in_channels=3, context_dim=1024,
                             roll_out=True, pooling_ctx_dim=768)
    m.randomize_zero_init_()
    m.to(dev).train()
    g = torch.Generator(device=dev).manual_seed(1)
    ctx = {"img_crossattn": torch.randn(B, M, 1024, device=dev, generator=g),
           "img_vector": torch.randn(B, 1024, device=dev, generator=g)}
    if m.xyz_cond:
        ctx["fps-xyz"] = torch.rand(B, N, 3, device=dev, generator=g) - 0.5
    return m, torch.randn(B, N, 3, device=dev, generator=g), ctx


def _timestep_embedding(t, dim=256, max_period=10000):
    """oracle/dit_oracle.timestep_embedding with its frequencies on t's device (the oracle builds them on the CPU)."""
    half = dim // 2
    freqs = torch.exp(-torch.log(torch.tensor(float(max_period))) * torch.arange(half, dtype=torch.float32) / half)
    args = t[:, None].float() * freqs.to(t.device)[None]
    return torch.cat([torch.cos(args), torch.sin(args)], dim=-1)


def stand_in(m):
    params = dict(m.named_parameters())
    return lambda x, t, context: dit_oracle.forward(params, x, t, context, m.num_heads, m.depth)


def step_fn(m, fn, x1, ctx, opt, transport):
    def step():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = transport.training_losses(fn, x1, dict(context=ctx))["loss"].mean()
        opt.zero_grad(set_to_none=True)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(m.parameters(), 1.0)
        opt.step()
    return step


def time_ms(fn, steps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(steps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / steps


def peak_mb(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def part15_bytes(B, D, Dc, Cout, K):
    """Bytes each Part 15 kernel's calls move in one step (fp32, 4 B)."""
    R, P = B * N, (B * N + 31) // 32
    return {
        "final_layer_bwd_kernel": 4 * (2 * R * D + R * Cout + P * (2 * D + Cout * D)),   # x read twice, dx, partials
        "embed_fc1_bwd_kernel": 4 * (2 * R * D + R * K + P * (D * K + D)),              # de1, x in, partials
        # adaLN (6D x D), t_embedder fc2 (D x D) and fc1 (D x 256), pooled projection (D x Dc): W read, dW written
        "linear_small_bwd_kernel": 4 * 2 * (6 * D * D + D * D + 256 * D + D * Dc),
        "layernorm_rows_bwd_kernel": 4 * 5 * B * Dc,
    }


def profile_kernels(step):
    from torch.profiler import ProfilerActivity, profile
    step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    times, launches = {}, 0
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            launches += 1
            times[ev.name] = times.get(ev.name, 0.0) + ev.device_time_total / 1000.0
    return launches, times


KERNELS = ("final_layer_bwd_kernel", "embed_fc1_bwd_kernel", "linear_small_bwd_kernel", "linear_small_dx_kernel",
           "layernorm_rows_bwd_kernel")


def ptxas():
    src = os.path.join(ROOT, "gaussiananything_b200", "csrc", "dit_model_grad.cu")
    nvcc = os.environ.get("NVCC") or "/usr/local/cuda/bin/nvcc"
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                            "-c", src, "-o", os.path.join(d, "o.o")], capture_output=True, text=True)
    out, name = {}, None
    for line in r.stderr.splitlines():
        mm = re.search(r"Compiling entry function '(\w+)'", line)
        if mm:
            name = next((k for k in KERNELS if k + "E" in mm.group(1)), mm.group(1))
        mm = re.search(r"(\d+) bytes spill stores", line)
        if mm and name:
            out.setdefault(name, {})["spill_stores"] = int(mm.group(1))
        mm = re.search(r"Used (\d+) registers", line)
        if mm and name:
            out.setdefault(name, {})["registers"] = int(mm.group(1))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    name, watts = card()
    res = dict(card=name, power_limit_w=watts, steps=a.steps, ptxas=ptxas(), configs={})
    print("card %s, power limit %s W" % (name, watts))
    transport = create_transport("Linear", "velocity")
    dit_oracle.timestep_embedding = _timestep_embedding
    for cfg in a.configs.split(","):
        arch, B = CONFIGS[cfg]
        m, x1, ctx = build(arch, B, dev)
        opt = torch.optim.AdamW(m.parameters(), lr=1e-4, weight_decay=0.05)
        ours = step_fn(m, functools.partial(dit_grad.model_forward, m), x1, ctx, opt, transport)
        ref = step_fn(m, stand_in(m), x1, ctx, opt, transport)
        r = dict(ours_ms=[], standin_ms=[])
        for _ in range(2):
            r["ours_ms"].append(time_ms(ours, a.steps))
            r["standin_ms"].append(time_ms(ref, a.steps))
        r["ours_peak_mb"], r["standin_peak_mb"] = peak_mb(ours), peak_mb(ref)
        r["ours_launches"], times = profile_kernels(ours)
        r["standin_launches"], _ = profile_kernels(ref)
        D, Cout = m.embed_dim, m.out_channels
        K = m.in_channels + (3 if m.xyz_cond and not m.use_pe_cond else 0)
        r["part15"] = {}
        for k, nbytes in part15_bytes(B, D, 1024, Cout, K).items():
            t = sum(v for n, v in times.items() if k in n)
            r["part15"][k] = dict(ms=t, floor_ms=nbytes / HBM * 1e3)
        print(cfg, json.dumps(r))
        res["configs"][cfg] = r
        del m, opt, ours, ref
        torch.cuda.empty_cache()
    print(json.dumps(res["ptxas"]))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
