"""Time LPIPS (VGG) and SSIM on the GPU and write the profile:

    python tools/lpips_leg.py [--out profiles/lpips_h100.md]

At 512^2 with random weights (oracle.lpips_oracle.random_state_dict; timing does not depend on the values):
- LPIPS for 16 pairs and for 1 pair through lpips.LPIPS (graph replay per chunk of 8 pairs), end to end;
- every kernel of one 8-pair chunk, launched alone: the 13 ReLU convolutions with their TFLOP/s (operations from the
  layer shapes, lpips_flops below), and the pack, pool, head and SSIM kernels with the bytes they must move over their
  time, against 3.35 TB/s;
- two stand-ins on the same card for the same 16 pairs: the fp32 cuDNN restatement (NCHW, TF32 off: the reference's
  precision) and a bf16 channels-last cuDNN restatement (the fair one), both features plus the torch head;
- SSIM for 16 pairs.
Device events around >= 0.3 s of back-to-back calls after a warm-up.  The card name and power limit are read in the
same run.  Needs a CUDA device.
"""
import argparse
import ctypes as C
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.dino_leg import card, time_replay  # noqa: E402

HBM = 3.35e12
BF16_PEAK = 989e12
SIZE = 512
SECONDS = 0.3


def lpips_flops(H, W):
    """Operations (2 per multiply-add) of VGG16's 13 convolutions up to relu5_3 for one H x W image, with the real
    3 input channels of the first layer: [(layer name, h, w, Cin, Cout, flops)].  611 712 per pixel at H, W % 16 == 0."""
    from gaussiananything_b200.lpips import CONVS
    out, h, w, tap = [], H, W, 0
    for k, i, cin, cout in CONVS:
        if k != tap:
            h, w, tap = h // 2, w // 2, k
        out.append(("features.%d" % i, h, w, cin, cout, 2 * 9 * cin * cout * h * w))
    return out


def torch_lpips(sd, a, b, dtype, channels_last):
    """Stand-in: the same network and head in eager torch (cuDNN convolutions)."""
    x = torch.cat([a, b], 0)
    shift = torch.tensor([-0.030, -0.088, -0.188], device=a.device).view(1, 3, 1, 1)
    scale = torch.tensor([0.458, 0.448, 0.450], device=a.device).view(1, 3, 1, 1)
    h = ((x - shift) / scale).to(dtype)
    if channels_last:
        h = h.contiguous(memory_format=torch.channels_last)
    n, val = a.shape[0], 0
    for k, (ws, bs, lin) in enumerate(sd):
        if k:
            h = F.max_pool2d(h, 2, 2)
        for w, bb in zip(ws, bs):
            h = F.relu(F.conv2d(h, w, bb, padding=1))
        f = h.float()
        f = f / (f.pow(2).sum(1, keepdim=True).sqrt() + 1e-10)
        val = val + ((f[:n] - f[n:]) ** 2 * lin).sum(1).mean((1, 2))
    return val


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "lpips_h100.md"))
    args = ap.parse_args()
    from gaussiananything_b200 import _lib, lpips
    from gaussiananything_b200._launch import ptr, stream
    from oracle.lpips_oracle import random_state_dict
    dev = torch.device("cuda:0")
    name, watts = card()
    sd = random_state_dict(0)
    model = lpips.LPIPS(state_dict=sd, device=dev)
    g = torch.Generator(device=dev).manual_seed(0)
    a16 = torch.rand(16, 3, SIZE, SIZE, generator=g, device=dev) * 2 - 1
    b16 = (a16 + 0.1 * torch.randn(a16.shape, generator=g, device=dev)).clamp(-1, 1)
    res = {"card": name, "power_limit_w": watts}
    flops = sum(f[-1] for f in lpips_flops(SIZE, SIZE))
    with torch.no_grad():
        for n in (16, 1):
            ms, _ = time_replay(lambda: model(a16[:n], b16[:n]), SECONDS)
            res["lpips_%d_pairs_ms" % n] = ms
            res["lpips_%d_pairs_tflops" % n] = 2 * n * flops / (ms * 1e-3) / 1e12
        # stand-ins on the same 16 pairs, and their agreement with the library's value
        for tag, dtype, cl in (("cudnn_fp32", torch.float32, False), ("cudnn_bf16_cl", torch.bfloat16, True)):
            tf32 = torch.backends.cudnn.allow_tf32
            torch.backends.cudnn.allow_tf32 = False
            torch.backends.cudnn.benchmark = True
            wsd = []
            for k, idx in enumerate(lpips.SLICES):
                ws = [sd["net.slice%d.%d.weight" % (k + 1, i)].to(dev, dtype) for i in idx]
                bs = [sd["net.slice%d.%d.bias" % (k + 1, i)].to(dev, dtype) for i in idx]
                wsd.append((ws, bs, sd["lin%d.model.1.weight" % k].to(dev).reshape(1, -1, 1, 1)))
            run = lambda: torch_lpips(wsd, a16[:8], b16[:8], dtype, cl)
            ms8, _ = time_replay(run, SECONDS)
            res[tag + "_16_pairs_ms"] = 2 * ms8                  # two chunks of 8, as the library runs them
            v = torch.cat([torch_lpips(wsd, a16[s:s + 8], b16[s:s + 8], dtype, cl) for s in (0, 8)])
            res[tag + "_max_abs_diff_vs_library"] = float((v - model(a16, b16).reshape(-1)).abs().max())
            torch.backends.cudnn.allow_tf32 = tf32
        res["ssim_16_pairs_ms"], _ = time_replay(lambda: lpips.ssim((a16 + 1) / 2, (b16 + 1) / 2), SECONDS)

        # per-kernel times for one chunk of 8 pairs (16 images)
        L, st = _lib.lib(), stream(dev)
        n = 8
        a, b = a16[:n].contiguous(), b16[:n].contiguous()
        x = torch.empty(2 * n, SIZE, SIZE, 8, device=dev, dtype=torch.bfloat16)
        kern = []
        ms, _ = time_replay(lambda: L.ga_lpips_pack(ptr(a), ptr(b), n, SIZE, SIZE, 0, ptr(model.shift),
                                                    ptr(model.scale), ptr(x), st), SECONDS)
        kern.append(("pack", ms, None, 2 * n * SIZE * SIZE * (3 * 4 + 16)))
        h = w = SIZE
        tap = 0
        partial = torch.empty(5, n, lpips.HEAD_BLOCKS, device=dev)
        for cv, (lname, _, _, cin, cout, fl) in zip(model.convs, lpips_flops(SIZE, SIZE)):
            if cv["tap"] != tap:
                y = torch.empty(2 * n, h // 2, w // 2, x.shape[-1], device=dev, dtype=torch.bfloat16)
                c = x.shape[-1]
                ms, _ = time_replay(lambda: L.ga_maxpool2x2_bf16(ptr(x), 2 * n, h, w, c, ptr(y), st), SECONDS)
                kern.append(("pool %dx%dx%d" % (h, w, c), ms, None, 2 * n * (h * w + (h // 2) * (w // 2)) * c * 2))
                x, h, w, tap = y, h // 2, w // 2, cv["tap"]
            y = torch.empty(2 * n, h, w, cv["cout"], device=dev, dtype=torch.bfloat16)
            ms, _ = time_replay(lambda: L.ga_conv3x3_relu_bf16(ptr(x), 2 * n, h, w, cv["cin"], ptr(cv["w"]), cv["kp"],
                                                               ptr(cv["b"]), cv["cout"], ptr(y), st), SECONDS)
            kern.append(("conv %s %dx%d %d->%d" % (lname, h, w, cin, cout), ms, 2 * n * fl, None))
            x = y
            if cv["last"]:
                c = cv["cout"]
                ms, _ = time_replay(lambda: L.ga_lpips_head(ptr(x), n, h, w, c, ptr(model.lin[tap]),
                                                            ptr(partial[tap]), st), SECONDS)
                kern.append(("head tap %d %dx%dx%d" % (tap, h, w, c), ms, None, 2 * n * h * w * c * 2))
        s0, s1 = (a + 1) / 2, (b + 1) / 2
        ms, _ = time_replay(lambda: lpips.ssim(s0, s1), SECONDS)
        kern.append(("ssim (call, 8 pairs)", ms, None, 2 * n * 3 * SIZE * SIZE * 4))
    res["kernels_8_pairs"] = [{"kernel": k, "us": ms * 1e3,
                               "tflops": (fl / (ms * 1e-3) / 1e12) if fl else None,
                               "tb_s": (by / (ms * 1e-3) / 1e12) if by else None} for k, ms, fl, by in kern]
    conv_ms = sum(ms for k, ms, fl, _ in kern if fl)
    res["conv_sum_8_pairs_ms"] = conv_ms
    print(json.dumps(res))
    lines = ["# LPIPS (VGG16) and SSIM at 512^2 on %s, power limit %s W" % (name, watts), "",
             "Written by `tools/lpips_leg.py` (random weights; device events around >= %.1f s of calls after a warm-up)."
             % SECONDS, "", "| measurement | value |", "|---|---|"]
    for k, v in res.items():
        if k != "kernels_8_pairs":
            lines.append("| %s | %s |" % (k, ("%.4g" % v) if isinstance(v, float) else v))
    lines += ["", "Per kernel, one chunk of 8 pairs (16 images), each kernel launched alone:", "",
              "| kernel | us | TFLOP/s (share of 989 bf16) | TB/s (share of 3.35) |", "|---|---|---|---|"]
    for r in res["kernels_8_pairs"]:
        tf = "%.1f (%.0f %%)" % (r["tflops"], 100 * r["tflops"] * 1e12 / BF16_PEAK) if r["tflops"] else ""
        bw = "%.2f (%.0f %%)" % (r["tb_s"], 100 * r["tb_s"] * 1e12 / HBM) if r["tb_s"] else ""
        lines.append("| %s | %.1f | %s | %s |" % (r["kernel"], r["us"], tf, bw))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
