"""CPU references of the LPIPS backward (include/ga_b200.h Part 9, gaussiananything_b200/lpips.py LPIPSLoss).

lpips_grad(sd, in0, in1, g, ...) is d(sum_i g_i LPIPS_i) / d in0 and / d in1:
  fp64          torch autograd through oracle/lpips_oracle.py's fp64 path.
  emulate_bf16  a hand-written backward that rounds where the kernels round, on the activations of the bf16-emulating
                forward (bf16 ReLU outputs, bf16 weights): the head gradient in fp32 with the zero-vector rule, the
                pool's routed gradient plus the head gradient summed in fp32, the ReLU mask as a select and one bf16
                rounding; masked dgrad convolutions in fp32 rounded once to bf16; the first conv of slices 1-4 to the
                pooled map in fp32; the input gradient in fp32.  The yardstick of the GPU tests.
"""
import torch
import torch.nn.functional as F

from oracle import lpips_oracle as lo

SLICES = lo.SLICES


def _bf16(t):
    return t.to(torch.bfloat16).to(t.dtype)


def _convs(sd):
    """[(slice k, weight, bias)] of the 13 convolutions in order."""
    return [(k, sd["net.slice%d.%d.weight" % (k + 1, i)], sd["net.slice%d.%d.bias" % (k + 1, i)])
            for k, idx in enumerate(SLICES) for i in idx]


def emulated_activations(sd, in0, in1, normalize=False):
    """The 13 ReLU outputs [2N, C, h, w] of oracle.lpips_oracle.features(..., emulate_bf16=True), fp32 holding bf16."""
    x = torch.cat([torch.as_tensor(in0), torch.as_tensor(in1)], 0).float()
    shift = sd.get("scaling_layer.shift", torch.tensor(lo.SHIFT)).reshape(1, 3, 1, 1).float()
    scale = sd.get("scaling_layer.scale", torch.tensor(lo.SCALE)).reshape(1, 3, 1, 1).float()
    if normalize:
        x = 2 * x - 1
    h = _bf16((x - shift) / scale)
    acts, tap = [], 0
    for k, w, b in _convs(sd):
        if k != tap:
            h, tap = F.max_pool2d(h, 2, 2), k
        h = _bf16(F.relu(F.conv2d(h, _bf16(w.float()), b.float(), padding=1)))
        acts.append(h)
    return acts


def head_grad(f, f_other, lin_w, g):
    """The tap's head gradient for the side whose features are f (fp32 [n, C, h, w]), as ga_lpips_tap_backward states
    it, in fp32: s (u / nf - (f / r) q), 0 where r = 0.  Its channel sums run in torch's order, not the kernel's."""
    h, w = f.shape[-2:]
    r = f.pow(2).sum(1, keepdim=True).sqrt()
    n0, n1 = r + 1e-10, f_other.pow(2).sum(1, keepdim=True).sqrt() + 1e-10
    u = 2 * (lin_w.float().reshape(1, -1, 1, 1) * (f / n0 - f_other / n1))
    S = (u * f).sum(1, keepdim=True)
    s = g.float().reshape(-1, 1, 1, 1) / float(h * w)
    q = (S / n0) / n0
    return torch.where(r > 0, s * (u / n0 - (f / r) * q), torch.zeros(()))


def pool_backward(y, dpool):
    """torch's max_pool2d(2, 2) backward: dpool to each window's first maximum of y in row-major order."""
    y = y.detach().clone().requires_grad_(True)
    return torch.autograd.grad(F.max_pool2d(y, 2, 2), y, dpool)[0]


def _emulated_side(sd, acts, side, g, normalize):
    n = len(g)
    convs = _convs(sd)
    mine = lambda t: t[side * n:(side + 1) * n]
    grad, dpool = None, None
    for j in range(len(convs) - 1, -1, -1):
        k, w, _ = convs[j]
        last = j + 1 == len(convs) or convs[j + 1][0] != k
        if last:
            f = acts[j]
            head = head_grad(mine(f), f[(1 - side) * n:(2 - side) * n], sd["lin%d.model.1.weight" % k], g)
            total = head if dpool is None else pool_backward(mine(f), dpool) + head
            grad = _bf16(torch.where(mine(f) > 0, total, torch.zeros(())))
        wb = _bf16(w.float())
        if j == 0:
            scale = sd.get("scaling_layer.scale", torch.tensor(lo.SCALE)).reshape(1, 3, 1, 1).float()
            dx = F.conv_transpose2d(grad, wb, padding=1) / scale
            return 2 * dx if normalize else dx
        dg = F.conv_transpose2d(grad, wb, padding=1)
        if convs[j - 1][0] == k:
            grad = _bf16(torch.where(mine(acts[j - 1]) > 0, dg, torch.zeros(())))
        else:
            dpool, grad = dg, None


def lpips_grad(sd, in0, in1, g, normalize=False, emulate_bf16=False, sides=(0, 1)):
    """[d/d in0, d/d in1] of sum_i g_i LPIPS_i (None for a side not in `sides`): fp64, or fp32 under emulate_bf16."""
    g = torch.as_tensor(g)
    if emulate_bf16:
        acts = emulated_activations(sd, in0, in1, normalize)
        return [_emulated_side(sd, acts, s, g, normalize) if s in sides else None for s in range(2)]
    x = [torch.as_tensor(t).double().detach().clone().requires_grad_(s in sides) for s, t in enumerate((in0, in1))]
    val = lo.lpips(sd, x[0], x[1], normalize=normalize)["value"]
    want = [x[s] for s in sides]
    got = torch.autograd.grad((val * g.double()).sum(), want)
    out = [None, None]
    for s, d in zip(sides, got):
        out[s] = d
    return out


def emulated_autograd(sd, in0, in1, g, normalize=False):
    """[d/d in0, d/d in1] by torch autograd through oracle.lpips_oracle's bf16-emulating forward: its casts round the
    gradient to bf16 at each ReLU output and at the packed input, its head runs in fp64."""
    x = [torch.as_tensor(t).float().detach().clone().requires_grad_(True) for t in (in0, in1)]
    val = lo.lpips(sd, x[0], x[1], normalize=normalize, emulate_bf16=True)["value"]
    return list(torch.autograd.grad((val * torch.as_tensor(g).double()).sum(), x))


def rel_l2(got, want):
    """Relative L2 per image [N] (fp64)."""
    got, want = got.double().flatten(1), want.double().flatten(1)
    return (got - want).norm(dim=1) / want.norm(dim=1).clamp_min(1e-300)
