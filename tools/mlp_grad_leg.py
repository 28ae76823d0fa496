"""Forward + backward timing of the differentiable FusedMLP (include/ga_b200.h Part 13) at the reference's training
shapes, against torch with autograd: bf16 autocast (F.linear -> F.gelu -> F.linear, cuBLAS) and fp32.

    python tools/mlp_grad_leg.py [--json out.json] [--seconds 1.0] [--shapes DiT-L,SRT]

Device events around >= `seconds` of back-to-back calls after a warm-up; the card's name and power limit are read in
the same call.  A forward plus backward with every gradient costs 12 M D hidden FLOP (six GEMMs of 2 M D hidden).
Every GEMM of the step has the same FLOPs, so each backward GEMM's time is listed beside the forward TN GEMMs'
(fc1 with the GELU epilogue, fc2).  Peak memory is the allocator's high-water mark over one step, above what was
allocated before it (inputs and parameters).
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gaussiananything_b200 import mlp as MLP  # noqa: E402

# name: (rows M, D, hidden)
SHAPES = {
    "DiT-L": (3072, 1024, 4096),
    "DiT-B": (3072, 768, 3072),
    "decoder-block": (768, 768, 3072),
    "upsampler-6912": (6912, 768, 3072),
    "upsampler-30720": (30720, 768, 3072),
    "upsampler-98304": (98304, 768, 3072),
    "SRT": (768, 256, 1024),
}


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


def run_shape(M, D, Hd, seconds):
    dev = torch.device("cuda")
    torch.manual_seed(0)
    m = MLP.FusedMLP(D, 0.0, "gelu", Hd // D).to(dev)
    ref = [torch.nn.Parameter(p.detach().clone()) for p in m.parameters()]      # w1, b1, w2, b2
    x = torch.randn(M, D, device=dev, dtype=torch.bfloat16).requires_grad_(True)
    x32 = x.detach().float().requires_grad_(True)
    dy = torch.randn(M, D, device=dev, dtype=torch.bfloat16)
    dy32 = dy.float()

    def ours():
        y = m(x)
        y.backward(dy)

    def torch_step(xi, g, autocast):
        w1, b1, w2, b2 = ref
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            y = torch.nn.functional.linear(torch.nn.functional.gelu(torch.nn.functional.linear(xi, w1, b1)), w2, b2)
        y.backward(g)

    row = dict(M=M, D=D, hidden=Hd, tflop=12.0 * M * D * Hd / 1e12)
    for name, fn in (("library", ours), ("torch_bf16_autocast", lambda: torch_step(x, dy, True)),
                     ("torch_fp32", lambda: torch_step(x32, dy32, False))):
        ms = time_ms(fn, seconds)
        row[name] = dict(ms=ms, tflops=row["tflop"] / (ms / 1e3), peak_mb=peak_mb(fn))
    # the single GEMMs of the library's step, all 2 M D hidden FLOP
    w1b, w2b = MLP._pack(m.mlp[0].weight), MLP._pack(m.mlp[2].weight)
    b1, b2 = m.mlp[1].bias.detach(), m.mlp[3].bias.detach()
    xb = x.detach()
    h, z = MLP._fc1(xb, w1b, b1, keep_pre=True)
    dz = MLP._dgrad(dy, w2b, z=z)
    gemms = {
        "fwd fc1 TN, GELU epilogue": lambda: MLP._fc1(xb, w1b, b1, keep_pre=False),
        "fwd fc1 TN, keeps Z": lambda: MLP._fc1(xb, w1b, b1, keep_pre=True),
        "fwd fc2 TN": lambda: MLP._forward_linear(h, w2b, b2, torch.bfloat16),
        "dgrad dZ = dY W2 o gelu'": lambda: MLP._dgrad(dy, w2b, z=z),
        "dgrad dx = dZ W1": lambda: MLP._dgrad(dz, w1b),
        "wgrad dW2 = dY^T H": lambda: MLP._wgrad(dy, h),
        "wgrad dW1 = dZ^T x": lambda: MLP._wgrad(dz, xb),
    }
    gf = 2.0 * M * D * Hd / 1e12
    row["gemms"] = {k: dict(ms=(t := time_ms(f, seconds / 4)), tflops=gf / (t / 1e3)) for k, f in gemms.items()}
    row["gemms"]["bias grads db1 + db2"] = dict(ms=time_ms(lambda: (MLP._bgrad(dz), MLP._bgrad(dy)), seconds / 4),
                                               tflops=None)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    a = ap.parse_args()
    name, watts = card()
    print("card: %s, power limit %s W" % (name, watts))
    rows = {}
    for s in a.shapes.split(","):
        rows[s] = run_shape(*SHAPES[s], a.seconds)
        r = rows[s]
        print("\n%s  M %d D %d hidden %d  (%.3f TFLOP per step)" % (s, r["M"], r["D"], r["hidden"], r["tflop"]))
        for k in ("library", "torch_bf16_autocast", "torch_fp32"):
            print("  %-22s %9.3f ms  %7.1f TFLOP/s  peak %8.1f MB" % (k, r[k]["ms"], r[k]["tflops"], r[k]["peak_mb"]))
        for k, v in r["gemms"].items():
            print("    %-28s %8.3f ms  %s" % (k, v["ms"], "" if v["tflops"] is None else "%6.1f TFLOP/s" % v["tflops"]))
        torch.cuda.empty_cache()
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(dict(card=name, power_limit_w=watts, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
