"""PatchGAN discriminator timings on one GPU (profiles/disc_h100.md): the g-step (16 images, gradient to the images,
parameters frozen), the d-step (16 reals then 16 fakes, hinge loss, gradients to the parameters) and the eval forward,
at 512^2, on the library, on fp32 cuDNN autograd and on bf16 channels-last cuDNN autocast, alternated in one run and
timed with CUDA events after a warm-up of every shape.  Prints one JSON line.

    python tools/disc_leg.py [--n 16] [--size 512] [--reps 10]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.nn as nn  # noqa: E402

from gaussiananything_b200 import disc  # noqa: E402


def torch_patchgan():
    c = disc.CHANNELS
    return nn.Sequential(
        nn.Conv2d(c[0], c[1], 4, 2, 1), nn.LeakyReLU(0.2, True),
        nn.Conv2d(c[1], c[2], 4, 2, 1, bias=False), nn.BatchNorm2d(c[2]), nn.LeakyReLU(0.2, True),
        nn.Conv2d(c[2], c[3], 4, 2, 1, bias=False), nn.BatchNorm2d(c[3]), nn.LeakyReLU(0.2, True),
        nn.Conv2d(c[3], c[4], 4, 1, 1, bias=False), nn.BatchNorm2d(c[4]), nn.LeakyReLU(0.2, True),
        nn.Conv2d(c[4], c[5], 4, 1, 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=16)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--kernels", action="store_true", help="per-kernel device times of the library (torch.profiler)")
    a = ap.parse_args()
    dev = "cuda:0"
    sd = disc.random_state_dict(1)
    lib = disc.NLayerDiscriminator()
    lib.load_state_dict(sd)
    lib = lib.to(dev).train()
    f32 = torch_patchgan()
    f32.load_state_dict({k[5:]: v for k, v in sd.items()})
    f32 = f32.to(dev).train()
    b16 = torch_patchgan()
    b16.load_state_dict({k[5:]: v for k, v in sd.items()})
    b16 = b16.to(dev).to(memory_format=torch.channels_last).train()
    torch.backends.cudnn.benchmark = True
    g = torch.Generator(device=dev).manual_seed(0)
    real = torch.rand(a.n, 3, a.size, a.size, device=dev, generator=g) * 2 - 1
    fake = (real + 0.1 * torch.randn(real.shape, device=dev, generator=g)).contiguous()

    def gstep(m, amp):
        for p in m.parameters():
            p.requires_grad_(False)
        x = fake.clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
            x_in = x.contiguous(memory_format=torch.channels_last) if amp else x
            loss = -m(x_in).float().mean()
        loss.backward()
        for p in m.parameters():
            p.requires_grad_(True)
        return x.grad

    def dstep(m, amp):
        for p in m.parameters():
            p.grad = None
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
            xr = real.contiguous(memory_format=torch.channels_last) if amp else real
            xf = fake.contiguous(memory_format=torch.channels_last) if amp else fake
            lr, lf = m(xr).float(), m(xf).float()
        (0.5 * (torch.relu(1.0 - lr).mean() + torch.relu(1.0 + lf).mean())).backward()
        return [p.grad for p in m.parameters()]

    def evalf(m, amp):
        m.eval()
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
            out = m(real.contiguous(memory_format=torch.channels_last) if amp else real).float()
        m.train()
        return out

    if a.kernels:
        return kernel_table(a, {"g_step": lambda: gstep(lib, False), "d_step": lambda: dstep(lib, False),
                                "eval_forward": lambda: evalf(lib, False)})

    impls = {"library": (lib, False), "cudnn_fp32": (f32, False), "cudnn_bf16_cl": (b16, True)}
    work = {"g_step": gstep, "d_step": dstep, "eval_forward": evalf}
    flops = disc.disc_flops(a.n, a.size, a.size)
    res = {}
    outs = {}
    for wname, fn in work.items():
        for iname, (m, amp) in impls.items():
            outs[(wname, iname)] = fn(m, amp)             # warm-up of every shape
    torch.cuda.synchronize()
    times = {k: [] for k in outs}
    peaks = {}
    for r in range(a.reps):
        for wname, fn in work.items():
            for iname, (m, amp) in impls.items():
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn(m, amp)
                e1.record()
                e1.synchronize()
                times[(wname, iname)].append(e0.elapsed_time(e1))
                peaks[(wname, iname)] = (torch.cuda.max_memory_allocated() - base) / 1e9
    for (wname, iname), ts in times.items():
        ts = sorted(ts)
        res["%s/%s" % (wname, iname)] = {"median_ms": ts[len(ts) // 2], "min_ms": ts[0], "peak_extra_gb": peaks[(wname, iname)]}
    # gradient differences of the library to both stand-ins (g-step: the images; d-step: every parameter)
    gl, gf, gb = outs[("g_step", "library")], outs[("g_step", "cudnn_fp32")], outs[("g_step", "cudnn_bf16_cl")]
    rel = lambda x, y: float((x.float() - y.float()).norm() / y.float().norm())
    res["grad_rel_l2"] = {"g_step_vs_fp32": rel(gl, gf), "g_step_bf16_vs_fp32": rel(gb, gf)}
    dl, df, db = outs[("d_step", "library")], outs[("d_step", "cudnn_fp32")], outs[("d_step", "cudnn_bf16_cl")]
    res["grad_rel_l2"]["d_step_vs_fp32_worst"] = max(rel(x, y) for x, y in zip(dl, df))
    res["grad_rel_l2"]["d_step_bf16_vs_fp32_worst"] = max(rel(x, y) for x, y in zip(db, df))
    res["forward_flops"] = flops
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True).stdout.strip()
    except OSError:
        q = torch.cuda.get_device_name(0)
    res["gpu"] = q
    res["n"], res["size"] = a.n, a.size
    print(json.dumps(res))


def conv_flops(N, H, W):
    """{category: FLOP} of the library's implicit-GEMM work: the forward of convs 1-4, their dgrad (convs 2-4), their
    weight gradients (convs 1-4), and conv 5."""
    sz = disc.sizes(H, W)
    c = disc.CHANNELS
    per = [2 * N * sz[k + 1][0] * sz[k + 1][1] * c[k] * c[k + 1] * 16 for k in range(5)]
    return {"fwd": sum(per[:4]), "dgrad": sum(per[1:4]), "wgrad": sum(per[:4]), "conv5": per[4]}


def kernel_table(a, work):
    """Device time per kernel name per call, summed over `reps` calls of each workload, and TFLOP/s of the GEMM
    groups (forward / dgrad / wgrad by template arguments: 4x4 with the LeakyReLU or stats epilogue is the forward,
    the LeakyReLU-grad and BN-grad epilogues and the 2x2 parity kernels are the dgrad)."""
    from torch.profiler import ProfilerActivity, profile
    fl = conv_flops(a.n, a.size, a.size)
    out = {}
    for name, fn in work.items():
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.reps):
                fn()
            torch.cuda.synchronize()
        rows = {}
        for ev in prof.key_averages():
            t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            if t > 0:
                rows[ev.key] = rows.get(ev.key, 0.0) + t / 1e3 / a.reps
        total = sum(rows.values())
        groups = {"fwd": 0.0, "dgrad": 0.0, "wgrad": 0.0, "conv5": 0.0}
        for k, ms in rows.items():
            if "wgrad_kernel" in k:
                groups["wgrad"] += ms
            elif "conv_igemm_kernel" in k:
                epi = k.split("ILi")[1] if "ILi" in k else ""
                groups["dgrad" if ("ELi4EE" in k or "ELi6EE" in k or k.startswith("void (anonymous namespace)::conv_igemm_kernel<2")
                                   or "ILi2E" in k) else "fwd"] += ms
            elif "disc_conv5" in k:
                groups["conv5"] += ms
        rate = {}
        calls = {"g_step": (1, 1, 0), "d_step": (2, 2, 2), "eval_forward": (1, 0, 0)}[name]
        for g, n_call in zip(("fwd", "dgrad", "wgrad"), calls):
            if groups[g] > 0:
                rate[g] = "%.1f TFLOP/s" % (n_call * fl[g] / (groups[g] * 1e-3) / 1e12)
        out[name] = {"total_kernel_ms": total, "groups_ms": groups, "gemm_rate": rate,
                     "kernels_ms": dict(sorted(rows.items(), key=lambda kv: -kv[1])[:25])}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
