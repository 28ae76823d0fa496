"""Forward + backward timing of memory_efficient_attention (include/ga_b200.h Part 12) at the reference's training
shapes, against every torch bf16 scaled_dot_product_attention backend that runs there (flash, memory-efficient,
cuDNN) and xformers when it is importable.

    python tools/attention_grad_leg.py [--json out.json] [--seconds 1.0]

Device events around >= `seconds` of back-to-back calls after a warm-up.  The card's name, power limit and maximum SM
clock are read in the same call.  Algorithmic FLOPs: 4 Nq Nk d per (sequence, head) for the forward and 10 Nq Nk d
for the backward (S, dP, dV, dK, dQ); the library's backward also forms S and dP a second time (once in the dK/dV
kernel, once in the dQ kernel), 4 Nq Nk d more, reported as `recompute_tflop`.  Inputs arrive as the reference
passes them: BMHK `unbind` views of a packed qkv, or BMK [B*H, N, d]; SDPA gets the same data transposed to
[B, H, N, d] views.  The library reads its operands in place, so it has no pack step; `pack_ms` is what packing
q, k, v, dO into head-major tensors and unpacking dq, dk, dv would cost (one copy per tensor), the alternative it
avoids.
"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gaussiananything_b200 import attention as A  # noqa: E402

# name: (B, H, Nq, Nk, d, layout); BMK shapes fold heads into the batch as the reference's 3-D callers do
SHAPES = {
    "dit_l_self_768": (8, 16, 768, 768, 64, "bmhk"),
    "dit2_b_self_768": (8, 12, 768, 768, 64, "bmhk"),
    "cross_dino_768x1369": (8 * 16, 1, 768, 1369, 64, "bmk"),
    "cross_clip_768x77": (8 * 16, 1, 768, 77, 64, "bmk"),
    "srt_agg_ca_768x32768": (8, 1, 768, 32768, 64, "bmk"),
    "vae_enc_mid_32768": (8, 1, 32768, 32768, 64, "bmk"),
    "vae_enc_view_4096": (64, 1, 4096, 4096, 64, "bmk"),
    "srt_self_768_d32": (8, 8, 768, 768, 32, "bmhk"),
    "upsampler_9tok": (768, 12, 9, 9, 64, "bmhk"),
    "upsampler_5tok": (6144, 12, 5, 5, 64, "bmhk"),
    "upsampler_4tok": (24576, 12, 4, 4, 64, "bmhk"),
    "short_cutover_17tok": (768, 12, 17, 17, 64, "bmhk"),
}

# An illegal memory access surfaced at this shape in one run of this script.  Every library call of a row is fenced by
# a device synchronise (the warm-up's, time_ms's and peak_mb's) before the first SDPA call, so a fault of a library
# kernel would have surfaced in the library's own row; it surfaced after the torch SDPA backends had run, so one of
# them raised it.  They are not run here again.  The library's results at this shape and layout are checked by
# tests/test_attention_grad_gpu.py (test_training_shapes, test_unbind_views_and_nan_padding).
BASELINE_NOT_RUN = {"upsampler_4tok": "a torch SDPA backend raised an illegal memory access at this shape; see the "
                                      "note above BASELINE_NOT_RUN"}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", "0"], capture_output=True, text=True, timeout=30)
        watts, mhz = (float(v) for v in r.stdout.strip().splitlines()[0].split(","))
    except Exception:
        watts = mhz = None
    return name, watts, mhz


def time_ms(fn, seconds):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    reps = max(3, math.ceil(seconds / max(e0.elapsed_time(e1) * 1e-3, 1e-6)))
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def peak_mb(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def make_inputs(B, H, Nq, Nk, d, layout, gen):
    dev = "cuda"
    if layout == "bmhk" and Nq == Nk:
        qkv = torch.randn(B, Nq, 3, H, d, generator=gen, device=dev).to(torch.bfloat16)
        q, k, v = qkv.unbind(2)
    elif layout == "bmhk":
        q = torch.randn(B, Nq, H, d, generator=gen, device=dev).to(torch.bfloat16)
        kv = torch.randn(B, Nk, 2, H, d, generator=gen, device=dev).to(torch.bfloat16)
        k, v = kv.unbind(2)
    else:
        q = torch.randn(B, Nq, d, generator=gen, device=dev).to(torch.bfloat16)
        k = torch.randn(B, Nk, d, generator=gen, device=dev).to(torch.bfloat16)
        v = torch.randn(B, Nk, d, generator=gen, device=dev).to(torch.bfloat16)
    do = torch.randn(q.shape, generator=gen, device=dev).to(torch.bfloat16)
    return [t.detach().requires_grad_(True) for t in (q, k, v)], do


def sdpa_fn(backend):
    from torch.nn.attention import sdpa_kernel

    def f(q, k, v):
        tr = (lambda t: t.transpose(1, 2)) if q.dim() == 4 else (lambda t: t.unsqueeze(1))
        with sdpa_kernel([backend]):
            o = torch.nn.functional.scaled_dot_product_attention(tr(q), tr(k), tr(v))
        return o.transpose(1, 2) if q.dim() == 4 else o.squeeze(1)
    return f


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--only", default=None, help="comma-separated shape names")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "attention_grad_leg needs a GPU"
    name, watts, mhz = card()
    res = {"card": name, "power_limit_w": watts, "max_sm_clock_mhz": mhz, "seconds_per_case": args.seconds,
           "cases": {}}
    from torch.nn.attention import SDPBackend
    impls = {"library": A.memory_efficient_attention,
             "sdpa_flash": sdpa_fn(SDPBackend.FLASH_ATTENTION),
             "sdpa_mem_efficient": sdpa_fn(SDPBackend.EFFICIENT_ATTENTION),
             "sdpa_cudnn": sdpa_fn(SDPBackend.CUDNN_ATTENTION)}
    try:
        import xformers.ops as xops
        impls["xformers"] = xops.memory_efficient_attention
        res["xformers"] = "measured"
    except Exception:
        res["xformers"] = "not measured: xformers is not importable here"
    names = args.only.split(",") if args.only else list(SHAPES)
    gen = torch.Generator(device="cuda").manual_seed(0)
    for case in names:
        B, H, Nq, Nk, d, layout = SHAPES[case]
        (q, k, v), do = make_inputs(B, H, Nq, Nk, d, layout, gen)
        pairs = B * H
        flop_f, flop_b = 4.0 * Nq * Nk * d * pairs, 10.0 * Nq * Nk * d * pairs
        row = {"shape": [B, H, Nq, Nk, d, layout], "fwd_tflop": flop_f / 1e12, "bwd_tflop": flop_b / 1e12,
               "recompute_tflop": 4.0 * Nq * Nk * d * pairs / 1e12, "impls": {}}
        for iname, fn in impls.items():
            def fwd():
                with torch.no_grad():
                    fn(q, k, v)

            def fwd_bwd():
                for t in (q, k, v):
                    t.grad = None
                fn(q, k, v).backward(do)
            if iname != "library" and case in BASELINE_NOT_RUN:
                row["impls"][iname] = {"error": "not measured: " + BASELINE_NOT_RUN[case]}
                continue
            try:
                fn(q, k, v).backward(do)
                torch.cuda.synchronize()
            except Exception as e:                      # a backend that does not take this shape
                row["impls"][iname] = {"error": "%s: %s" % (type(e).__name__, str(e).splitlines()[0][:160])}
                print("%-24s %s: %s" % (case, iname, row["impls"][iname]["error"]), flush=True)
                if "illegal memory access" in str(e):
                    raise
                continue
            tf, tfb = time_ms(fwd, args.seconds), time_ms(fwd_bwd, args.seconds)
            row["impls"][iname] = {"fwd_ms": tf, "fwd_bwd_ms": tfb, "bwd_ms": tfb - tf,
                                   "fwd_bwd_tflops": (flop_f + flop_b) / (tfb * 1e-3) / 1e12,
                                   "peak_mb": peak_mb(fwd_bwd)}

        def pack():
            packed = [t.detach().transpose(1, 2).contiguous() if t.dim() == 4 else t.detach().contiguous()
                      for t in (q, k, v, do)]
            for t in packed[:3]:
                t.transpose(1, 2).contiguous() if t.dim() == 4 else t.clone()
        row["pack_ms"] = 0.0
        row["pack_alternative_ms"] = time_ms(pack, args.seconds / 2)
        res["cases"][case] = row
        lib = row["impls"]["library"]
        if "fwd_bwd_ms" not in lib:
            print("%-24s library %s" % (case, lib), flush=True)
            continue
        best = min([(r["fwd_bwd_ms"], n) for n, r in row["impls"].items() if n != "library" and "fwd_bwd_ms" in r]
                   or [(float("nan"), "none")])
        print("%-24s library fwd %.3f ms fwd+bwd %.3f ms (%.0f TFLOP/s)  best other %s %.3f ms" % (
            case, lib["fwd_ms"], lib["fwd_bwd_ms"], lib["fwd_bwd_tflops"], best[1], best[0]), flush=True)
        del q, k, v, do
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
