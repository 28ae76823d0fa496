"""Time the LPIPS backward (LPIPSLoss, gradient to pred only) on the GPU and write the profile:

    python tools/lpips_grad_leg.py [--out profiles/lpips_grad_h100.md]

With random weights (oracle.lpips_oracle.random_state_dict; timing does not depend on the values):
- LPIPSLoss forward + backward for 16 pairs at 288^2 (the reference's training crop) and at 512^2, beside the
  forward alone (no grad, graph replay);
- every kernel of the backward of one chunk of 8 pairs at 512^2, launched alone: the dgrad convolutions with their
  TFLOP/s, the tap and input backward kernels with the bytes they must move over their time, against 3.35 TB/s;
- the launch gaps of one forward + backward at 288^2 from torch.profiler (kernel time against wall time);
- peak memory of forward + backward;
- two torch autograd stand-ins on the same frozen weights: bf16 channels-last cuDNN, and fp32 with TF32 off (the
  reference's precision), with their largest gradient difference from the library's.
Device events around >= 0.3 s of back-to-back calls after a warm-up.  The card name and power limit are read in the
same run.  Needs a CUDA device.
"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.dino_leg import card, time_replay  # noqa: E402
from tools.lpips_leg import lpips_flops  # noqa: E402

HBM = 3.35e12
BF16_PEAK = 989e12
SECONDS = 0.3


def torch_loss(wsd, pred, target, dtype, channels_last):
    """Stand-in: LPIPS(target, pred).mean() through eager torch autograd (cuDNN convolutions)."""
    x = torch.cat([target, pred], 0)
    shift = torch.tensor([-0.030, -0.088, -0.188], device=x.device).view(1, 3, 1, 1)
    scale = torch.tensor([0.458, 0.448, 0.450], device=x.device).view(1, 3, 1, 1)
    h = ((x - shift) / scale).to(dtype)
    if channels_last:
        h = h.contiguous(memory_format=torch.channels_last)
    n, val = pred.shape[0], 0
    for k, (ws, bs, lin) in enumerate(wsd):
        if k:
            h = F.max_pool2d(h, 2, 2)
        for w, bb in zip(ws, bs):
            h = F.relu(F.conv2d(h, w, bb, padding=1))
        f = h.float()
        f = f / (f.pow(2).sum(1, keepdim=True).sqrt() + 1e-10)
        val = val + ((f[:n] - f[n:]) ** 2 * lin).sum(1).mean((1, 2))
    return val.mean()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "lpips_grad_h100.md"))
    args = ap.parse_args()
    from gaussiananything_b200 import lpips
    from gaussiananything_b200._launch import ptr, stream
    from oracle.lpips_oracle import random_state_dict
    dev = torch.device("cuda:0")
    name, watts = card()
    sd = random_state_dict(0)
    model = lpips.LPIPS(state_dict=sd, device=dev)
    crit = lpips.LPIPSLoss(lpips=model)
    gen = torch.Generator(device=dev).manual_seed(0)
    res = {"card": name, "power_limit_w": watts}
    for S in (288, 512):
        tgt = torch.rand(16, 3, S, S, generator=gen, device=dev) * 2 - 1
        pred0 = (tgt + 0.1 * torch.randn(tgt.shape, generator=gen, device=dev)).clamp(-1, 1)
        pred = pred0.clone().requires_grad_(True)

        def fwd_bwd():
            pred.grad = None
            crit(pred, tgt).backward()
        with torch.no_grad():
            res["fwd_only_16_pairs_%d_ms" % S], _ = time_replay(lambda: crit(pred0, tgt), SECONDS)
        res["fwd_bwd_16_pairs_%d_ms" % S], _ = time_replay(fwd_bwd, SECONDS)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        fwd_bwd()
        torch.cuda.synchronize()
        res["peak_mem_above_inputs_16_pairs_%d_MB" % S] = (torch.cuda.max_memory_allocated(dev) - base) / 1e6
        mine = pred.grad.clone()
        for tag, dtype, cl in (("cudnn_fp32", torch.float32, False), ("cudnn_bf16_cl", torch.bfloat16, True)):
            tf32 = torch.backends.cudnn.allow_tf32
            torch.backends.cudnn.allow_tf32 = False
            torch.backends.cudnn.benchmark = True
            wsd = []
            for k, idx in enumerate(lpips.SLICES):
                ws = [sd["net.slice%d.%d.weight" % (k + 1, i)].to(dev, dtype) for i in idx]
                bs = [sd["net.slice%d.%d.bias" % (k + 1, i)].to(dev, dtype) for i in idx]
                wsd.append((ws, bs, sd["lin%d.model.1.weight" % k].to(dev).reshape(1, -1, 1, 1)))
            p2 = pred0.clone().requires_grad_(True)

            def run():
                p2.grad = None
                tot = 0
                for s in (0, 8):                             # two chunks of 8, as the library runs them
                    tot = tot + torch_loss(wsd, p2[s:s + 8], tgt[s:s + 8], dtype, cl) / 2
                tot.backward()
            res["%s_fwd_bwd_16_pairs_%d_ms" % (tag, S)], _ = time_replay(run, SECONDS)
            run()
            res["%s_max_grad_diff_vs_library_%d" % (tag, S)] = float((p2.grad - mine).abs().max())
            res["%s_grad_rel_l2_vs_library_%d" % (tag, S)] = float((p2.grad - mine).norm() / p2.grad.norm())
            torch.backends.cudnn.allow_tf32 = tf32
        res["library_max_abs_grad_%d" % S] = float(mine.abs().max())

    # launch gaps: one forward + backward at 288^2 under torch.profiler
    tgt = torch.rand(16, 3, 288, 288, generator=gen, device=dev) * 2 - 1
    pred = tgt.clone().add_(0.05).requires_grad_(True)
    from torch.profiler import ProfilerActivity, profile
    crit(pred, tgt).backward()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        pred.grad = None
        crit(pred, tgt).backward()
        torch.cuda.synchronize()
    ev = sorted([e for e in prof.events() if e.device_type.name == "CUDA" and e.device_time > 0],
                key=lambda e: e.time_range.start)
    if ev:
        span = ev[-1].time_range.end - ev[0].time_range.start
        busy = sum(e.device_time for e in ev)
        gaps = [b.time_range.start - a.time_range.end for a, b in zip(ev, ev[1:])]
        res["profile_288_kernels"] = len(ev)
        res["profile_288_span_us"] = span
        res["profile_288_kernel_busy_us"] = busy
        res["profile_288_median_gap_us"] = sorted(gaps)[len(gaps) // 2] if gaps else 0.0
        res["profile_288_max_gap_us"] = max(gaps) if gaps else 0.0

    # per-kernel times of one chunk's backward (8 pairs, pred side) at 512^2
    S, n = 512, 8
    a = torch.rand(n, 3, S, S, generator=gen, device=dev) * 2 - 1
    b = (a + 0.1 * torch.randn(a.shape, generator=gen, device=dev)).clamp(-1, 1)
    L, st = model.L, stream(dev)
    with torch.no_grad():
        saved = model._forward_saving(a, b, False, (1,))
        gv = torch.full((n,), 1.0 / n, device=dev)
        kern = []
        acts, taps = saved["acts"][1], saved["taps"]
        dpool = None
        for j in range(len(model.convs) - 1, -1, -1):
            cv = model.convs[j]
            k = cv["tap"]
            h, w = S >> k, S >> k
            if cv["last"]:
                grad = torch.empty(n, h, w, cv["cout"], device=dev, dtype=torch.bfloat16)
                c, dp = cv["cout"], dpool
                ms, _ = time_replay(lambda: L.ga_lpips_tap_backward(ptr(taps[k]), n, h, w, c, 1, ptr(model.lin[k]),
                                                                    ptr(gv), ptr(dp), ptr(grad), st), SECONDS)
                by = n * h * w * c * 2 * (3 if dp is not None else 2) + (n * h * w * c if dp is not None else 0) * 2 \
                    + n * h * w * c * 2
                kern.append(("tap backward %d %dx%dx%d%s" % (k, h, w, c, " + pool" if dp is not None else ""), ms,
                             None, by))
            fl = 2 * 9 * cv["cin"] * cv["cout"] * h * w * n
            if j == 0:
                dx = torch.empty(n, 3, S, S, device=dev)
                g0 = grad
                ms, _ = time_replay(lambda: L.ga_lpips_input_backward(ptr(g0), n, S, S, ptr(model.w0_flip),
                                                                      ptr(model.scale), 0, ptr(dx), st), SECONDS)
                kern.append(("input backward (features.0 dgrad + pack)", ms, None, n * S * S * (64 * 2 + 3 * 4)))
                break
            g_in = grad
            if model.convs[j - 1]["tap"] == k:
                out = torch.empty(n, h, w, cv["cin"], device=dev, dtype=torch.bfloat16)
                mk = acts[j - 1]
                ms, _ = time_replay(lambda: L.ga_conv3x3_mask_bf16(ptr(g_in), n, h, w, cv["cout"], ptr(cv["wf"]),
                                                                   cv["kpf"], cv["cin"], ptr(mk), ptr(out), st),
                                    SECONDS)
                kern.append(("dgrad+mask conv %d %dx%d %d->%d" % (j, h, w, cv["cout"], cv["cin"]), ms, fl, None))
                grad = out
            else:
                dpool = torch.empty(n, h, w, cv["cin"], device=dev)
                dp = dpool
                ms, _ = time_replay(lambda: L.ga_conv3x3_bf16(ptr(g_in), n, h, w, cv["cout"], ptr(cv["wf"]),
                                                              cv["kpf"], None, cv["cin"], 1, None, ptr(dp), None, st),
                                    SECONDS)
                kern.append(("dgrad conv %d to pooled map (fp32) %dx%d %d->%d" % (j, h, w, cv["cout"], cv["cin"]),
                             ms, fl, None))
    res["kernels_8_pairs_512"] = [{"kernel": kk, "us": ms * 1e3,
                                   "tflops": (fl / (ms * 1e-3) / 1e12) if fl else None,
                                   "tb_s": (by / (ms * 1e-3) / 1e12) if by else None} for kk, ms, fl, by in kern]
    res["bwd_kernel_sum_8_pairs_512_ms"] = sum(ms for _, ms, _, _ in kern)
    print(json.dumps(res))
    lines = ["# LPIPS (VGG16) backward on %s, power limit %s W" % (name, watts), "",
             "Written by `tools/lpips_grad_leg.py` (random weights; device events around >= %.1f s of calls after a "
             "warm-up).  LPIPSLoss with the gradient to pred only, 16 pairs." % SECONDS, "",
             "| measurement | value |", "|---|---|"]
    for k, v in res.items():
        if k != "kernels_8_pairs_512":
            lines.append("| %s | %s |" % (k, ("%.4g" % v) if isinstance(v, float) else v))
    lines += ["", "Backward kernels of one chunk of 8 pairs at 512^2 (pred side only), each launched alone:", "",
              "| kernel | us | TFLOP/s (share of 989 bf16) | TB/s (share of 3.35) |", "|---|---|---|---|"]
    for r in res["kernels_8_pairs_512"]:
        tf = "%.1f (%.0f %%)" % (r["tflops"], 100 * r["tflops"] * 1e12 / BF16_PEAK) if r["tflops"] else ""
        bw = "%.2f (%.0f %%)" % (r["tb_s"], 100 * r["tb_s"] * 1e12 / HBM) if r["tb_s"] else ""
        lines.append("| %s | %.1f | %s | %s |" % (r["kernel"], r["us"], tf, bw))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
