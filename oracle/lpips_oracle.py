"""CPU restatement of LPIPS (VGG16, version 0.1) and SSIM (include/ga_b200.h Part 8, gaussiananything_b200/lpips.py).

lpips(sd, in0, in1) runs in fp64 by default.  emulate_bf16=True restates what the GPU path rounds: the packed input
(x - shift) / scale computed in fp32 and rounded to bf16, the conv weights rounded to bf16, each convolution in
fp32 (bias included) with its ReLU output rounded to bf16, max pools on those bf16 values; the head and the means then
run in fp64 on the bf16 features.  That mode is the yardstick of the GPU tests.  ssim(...) is _ssim with
size_average=False in fp64, with the fp32 window values the GPU uses.
"""
import math

import torch
import torch.nn.functional as F

TAPS = 5
SLICES = ((0, 2), (5, 7), (10, 12, 14), (17, 19, 21), (24, 26, 28))
SHIFT = (-0.030, -0.088, -0.188)
SCALE = (0.458, 0.448, 0.450)


def _bf16(t):
    return t.to(torch.bfloat16).to(t.dtype)


def features(sd, in0, in1, normalize=False, emulate_bf16=False):
    """The five tap activations [2N, C, h, w] (in0's images first) in fp64, or fp32 holding bf16 values."""
    x = torch.cat([torch.as_tensor(in0), torch.as_tensor(in1)], 0)
    shift = sd.get("scaling_layer.shift", torch.tensor(SHIFT)).reshape(1, 3, 1, 1)
    scale = sd.get("scaling_layer.scale", torch.tensor(SCALE)).reshape(1, 3, 1, 1)
    if emulate_bf16:
        x = x.float()
        if normalize:
            x = 2 * x - 1
        h = _bf16((x - shift.float()) / scale.float())
    else:
        x = x.double()
        if normalize:
            x = 2 * x - 1
        h = (x - shift.double()) / scale.double()
    taps = []
    for k, idx in enumerate(SLICES):
        if k:
            h = F.max_pool2d(h, 2, 2)
        for i in idx:
            w, b = sd["net.slice%d.%d.weight" % (k + 1, i)], sd["net.slice%d.%d.bias" % (k + 1, i)]
            if emulate_bf16:
                h = _bf16(F.relu(F.conv2d(h, _bf16(w.float()), b.float(), padding=1)))
            else:
                h = F.relu(F.conv2d(h, w.double(), b.double(), padding=1))
        taps.append(h)
    return taps


def head(sd, taps, n):
    """Per-pair, per-tap spatial means [n, 5] and their sum [n] (fp64) from the tap activations."""
    per = []
    for k, f in enumerate(taps):
        f = f.double()
        f0, f1 = f[:n], f[n:]
        f0 = f0 / (f0.pow(2).sum(1, keepdim=True).sqrt() + 1e-10)
        f1 = f1 / (f1.pow(2).sum(1, keepdim=True).sqrt() + 1e-10)
        w = sd["lin%d.model.1.weight" % k].double().reshape(1, -1, 1, 1)
        per.append(((f0 - f1) ** 2 * w).sum(1).mean((1, 2)))
    per = torch.stack(per, 1)
    return per, per.sum(1)


def lpips(sd, in0, in1, normalize=False, emulate_bf16=False):
    """{'taps': [5 x [2N, C, h, w]], 'per_tap' [N, 5], 'value' [N]} (fp64 values)."""
    taps = features(sd, in0, in1, normalize, emulate_bf16)
    per, val = head(sd, taps, len(in0))
    return {"taps": taps, "per_tap": per, "value": val}


def gaussian_window(window_size=11, sigma=1.5):
    """create_window's 2D window [ws, ws] in fp32, as the reference computes it."""
    g = torch.tensor([math.exp(-(x - window_size // 2) ** 2 / float(2 * sigma ** 2)) for x in range(window_size)],
                     dtype=torch.float32)
    g = (g / g.sum()).unsqueeze(1)
    return g.mm(g.t()).float()


def ssim(img1, img2, window_size=11):
    """Per-image SSIM [N] in fp64 (zero padding, C1 = 0.01^2, C2 = 0.03^2, mean over C, H, W)."""
    a, b = torch.as_tensor(img1).double(), torch.as_tensor(img2).double()
    C = a.shape[1]
    w = gaussian_window(window_size).double().expand(C, 1, window_size, window_size).contiguous()
    conv = lambda t: F.conv2d(t, w, padding=window_size // 2, groups=C)
    mu1, mu2 = conv(a), conv(b)
    mu1_sq, mu2_sq, mu1_mu2 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    s1, s2, s12 = conv(a * a) - mu1_sq, conv(b * b) - mu2_sq, conv(a * b) - mu1_mu2
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    m = ((2 * mu1_mu2 + C1) * (2 * s12 + C2)) / ((mu1_sq + mu2_sq + C1) * (s1 + s2 + C2))
    return m.mean((1, 2, 3))


def random_state_dict(seed=0, bias_std=0.05, lin_hi=0.2):
    """The LPIPS layout with seeded random weights: Kaiming-normal convolutions (torchvision's VGG initialisation)
    with N(0, bias_std) biases, U(0, lin_hi) linear layers (the trained ones are non-negative), the scaling layer's
    constants.  For tests and benchmarks: the real weights are not fetched."""
    g = torch.Generator().manual_seed(seed)
    sd = {"scaling_layer.shift": torch.tensor(SHIFT).reshape(1, 3, 1, 1),
          "scaling_layer.scale": torch.tensor(SCALE).reshape(1, 3, 1, 1)}
    cin = 3
    for k, idx in enumerate(SLICES):
        cout = (64, 128, 256, 512, 512)[k]
        for i in idx:
            std = math.sqrt(2.0 / (cout * 9))                       # kaiming_normal_, fan_out, relu
            sd["net.slice%d.%d.weight" % (k + 1, i)] = torch.randn(cout, cin, 3, 3, generator=g) * std
            sd["net.slice%d.%d.bias" % (k + 1, i)] = torch.randn(cout, generator=g) * bias_std
            cin = cout
        sd["lin%d.model.1.weight" % k] = torch.rand(1, cout, 1, 1, generator=g) * lin_hi
    return sd
