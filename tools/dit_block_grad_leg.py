"""Forward + backward timing of the trainable DiT block (include/ga_b200.h Part 14, gaussiananything_b200/dit_grad.py)
against the torch stand-in: oracle/dit_oracle.block_forward under bf16 autocast (cuBLAS GEMMs, SDPA attention) with
autograd.

    python tools/dit_block_grad_leg.py [--json out.json] [--seconds 2.0]

Device events around >= `seconds` of back-to-back steps (forward, then backward of every gradient: x, t, context and
the 21 parameters) after a warm-up; the card's name and power limit are read in the same call.  Peak memory is the
allocator's high-water mark over one step above what was allocated before it.  A separate profiled step gives the
launch count and each Part 14 kernel's time, listed beside its byte floor at 3.35 TB/s (the bytes its calls in one
step must move, from the shapes).
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gaussiananything_b200 import dit, dit_grad  # noqa: E402
from oracle import dit_oracle  # noqa: E402

# name: (B, N, M, D, heads, Dc)
SHAPES = {"DiT-L": (4, 768, 1369, 1024, 16, 1024), "DiT-B": (4, 2048, 1369, 768, 12, 1024)}
HBM = 3.35e12


def card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        watts = float(r.stdout.strip().splitlines()[0])
    except Exception:
        watts = None
    return name, watts


def time_ms(fn, seconds):
    fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    torch.cuda.synchronize()
    n = max(3, int(seconds * 1000.0 / max(s.elapsed_time(e), 1e-3)))
    s.record()
    for _ in range(n):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / n


def peak_mb(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def row_kernel_bytes(B, N, M, D):
    """Bytes each Part 14 kernel's calls move in one step (fp32 rows 4 B, bf16 2 B)."""
    R, RM = B * N, B * M
    P = (R + 31) // 32
    return {
        "rmsnorm_bwd_kernel": 3 * 16 * R * D,            # dh, x, dx_in read, dx written (norm2, norm1, prenorm)
        "gate_bwd_kernel": 2 * 10 * R * D,               # dy, a read, da (bf16) written
        "gate_residual_kernel": 2 * 14 * R * D + 12 * R * D,
        "qk_norm_fwd_kernel": 4 * D * (3 * R + RM),      # bf16 in and out: CA q, CA k, SA q|k
        "qk_norm_bwd_kernel": 6 * D * (3 * R + RM),      # pre-norm, dq/dk read, gradient written
        "partial_sum_kernel": 4 * 9 * P * D,             # the norm and modulation partials
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    ap.add_argument("--seconds", type=float, default=2.0)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    name, watts = card()
    out = dict(card=name, power_limit_w=watts, shapes={})
    for label, (B, N, M, D, H, Dc) in SHAPES.items():
        torch.manual_seed(0)
        blk = dit.ImageCondDiTBlockPixelArtRMSNormClayLRM(D, H, Dc).to(dev)
        x = torch.randn(B, N, D, device=dev, requires_grad=True)
        t = (0.3 * torch.randn(B, 6 * D, device=dev)).requires_grad_(True)
        c = torch.randn(B, M, Dc, device=dev, requires_grad=True)
        dy = torch.randn(B, N, D, device=dev)
        sd = dict(blk.named_parameters())

        def ours():
            blk(x, t, c).backward(dy)

        def standin():
            with torch.autocast("cuda", dtype=torch.bfloat16):
                y = dit_oracle.block_forward(sd, "", x, t, c, H)
            y.float().backward(dy)

        def ours_fwd():
            with torch.no_grad():
                blk(x, t, c)

        r = dict(B=B, N=N, M=M, D=D, heads=H, Dc=Dc)
        for _ in range(2):                                          # alternate, to see the spread
            r.setdefault("ours_ms", []).append(time_ms(ours, args.seconds))
            r.setdefault("standin_ms", []).append(time_ms(standin, args.seconds))
        r["ours_forward_nograd_ms"] = time_ms(ours_fwd, args.seconds)
        r["ours_peak_mb"], r["standin_peak_mb"] = peak_mb(ours), peak_mb(standin)
        from torch.profiler import ProfilerActivity, profile
        ours()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ours()
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in ev.name and "Memset" not in ev.name:
                k = kern.setdefault(ev.name, [0, 0.0])
                k[0] += 1
                k[1] += ev.device_time / 1000.0 if hasattr(ev, "device_time") else ev.cuda_time / 1000.0
        r["launches"] = sum(v[0] for v in kern.values())
        rows = {}
        for short, nbytes in row_kernel_bytes(B, N, M, D).items():
            hit = [(n, v) for n, v in kern.items() if short in n]
            ms = sum(v[1] for _, v in hit)
            rows[short] = dict(calls=sum(v[0] for _, v in hit), ms=ms, floor_ms=nbytes / HBM * 1e3,
                               share_of_floor=(nbytes / HBM * 1e3) / ms if ms else None)
        r["row_kernels"] = rows
        r["all_kernels_ms"] = {n: v for n, v in sorted(kern.items(), key=lambda kv: -kv[1][1])}
        out["shapes"][label] = r
        print("%s: ours %s ms, stand-in %s ms, launches %d, peak %.0f MB vs %.0f MB" % (
            label, ["%.3f" % v for v in r["ours_ms"]], ["%.3f" % v for v in r["standin_ms"]], r["launches"],
            r["ours_peak_mb"], r["standin_peak_mb"]))
        for k, v in rows.items():
            print("  %-22s %2d calls %8.1f us, floor %7.1f us" % (k, v["calls"], v["ms"] * 1e3, v["floor_ms"] * 1e3))
        del blk, x, t, c, dy, sd
        torch.cuda.empty_cache()
    print("card: %s, power limit %s W" % (name, watts))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
