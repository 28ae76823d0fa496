"""PatchGAN discriminator on the library's kernels (include/ga_b200.h Part 11).

  NLayerDiscriminator  mirrors the reference's nsr/losses/disc.py NLayerDiscriminator(input_nc=3, ndf=64, n_layers=3,
          use_actnorm=False), the pix2pix PatchGAN that E3DGE_with_AdvLoss builds for the VAE's adversarial loss: five
          4x4 convolutions with pad 1 (strides 2, 2, 2, 1, 1; channels 3 -> 64 -> 128 -> 256 -> 512 -> 1),
          BatchNorm2d after convolutions 2-4 and LeakyReLU(0.2) after convolutions 1-4.

The parameters live in real nn.Conv2d / nn.BatchNorm2d children of an nn.Sequential named `main`, so the state dict
is the reference's and weights_init, load_state_dict, .to(), optimisers and DDP see ordinary modules; their forward is
never called.  forward() runs one autograd Function over the input and every parameter: the input gradient is formed
only when the input requires grad, and a parameter's gradient only when that parameter requires grad.

Precision: bf16 operands and activations with fp32 accumulation, fp32 pre-normalisation outputs and logits, BatchNorm
statistics merged in fp64 (INTEGRATION.md section 3j).  Weights are repacked from the fp32 parameters on every call.
"""
import torch
import torch.nn as nn

from . import _launch, _lib
from ._launch import ptr as _p

INPUT_NC, NDF, N_LAYERS = 3, 64, 3
CHANNELS = (3, 64, 128, 256, 512, 1)
STRIDES = (2, 2, 2, 1, 1)
CONV_KEYS = ("main.0", "main.2", "main.5", "main.8", "main.11")
BN_KEYS = ("main.3", "main.6", "main.9")
SLOPE = 0.2


def out_size(h, stride):
    """torch's Conv2d output size for kernel 4, pad 1."""
    return (h + 2 - 4) // stride + 1


def sizes(H, W):
    """[(h, w)] of the input and of each convolution's output."""
    out = [(H, W)]
    for s in STRIDES:
        h, w = out[-1]
        out.append((out_size(h, s), out_size(w, s)))
    return out


def disc_flops(N, H, W):
    """Useful multiply-adds x 2 of one forward of N images of H x W (the convolutions; padding taps not removed)."""
    total = 0
    for k, (h, w) in enumerate(sizes(H, W)[1:]):
        total += 2 * N * h * w * CHANNELS[k] * CHANNELS[k + 1] * 16
    return total


def state_dict_shapes():
    """{key: shape} of the reference module's state dict (tests/golden/disc_keys.json)."""
    s = {}
    for k, key in enumerate(CONV_KEYS):
        s[key + ".weight"] = (CHANNELS[k + 1], CHANNELS[k], 4, 4)
        if k in (0, 4):
            s[key + ".bias"] = (CHANNELS[k + 1],)
    for k, key in enumerate(BN_KEYS):
        c = CHANNELS[k + 2]
        for name in ("weight", "bias", "running_mean", "running_var"):
            s["%s.%s" % (key, name)] = (c,)
        s[key + ".num_batches_tracked"] = ()
    return dict(sorted(s.items(), key=lambda kv: (int(kv[0].split(".")[1]), kv[0])))


def random_state_dict(seed):
    """Weights drawn as the reference's weights_init draws them: convolutions N(0, 0.02), BatchNorm weight N(1, 0.02)
    and bias 0; conv 1 and conv 5 biases N(0, 0.02) (the reference leaves Conv2d's default uniform init there).
    Running statistics 0 and 1, num_batches_tracked 0.  fp32, CPU."""
    g = torch.Generator().manual_seed(int(seed))
    sd = {}
    for key, shape in state_dict_shapes().items():
        name = key.rsplit(".", 1)[1]
        if key.rsplit(".", 1)[0] in CONV_KEYS:
            sd[key] = torch.randn(shape, generator=g) * 0.02
        elif name == "weight":
            sd[key] = 1.0 + torch.randn(shape, generator=g) * 0.02
        elif name in ("bias", "running_mean"):
            sd[key] = torch.zeros(shape)
        elif name == "running_var":
            sd[key] = torch.ones(shape)
        else:
            sd[key] = torch.zeros((), dtype=torch.long)
    return sd


# ---- weight packs (include/ga_b200.h Part 11)
def pack_forward(w, cin_pad):
    """bf16 [Co, kp]: column (ky * 4 + kx) * cin_pad + ci = W[co, ci, ky, kx]; kp = 16 cin_pad rounded up to 64."""
    co, ci = w.shape[:2]
    kp = _launch.round_up(16 * cin_pad, 64)
    out = torch.zeros(co, kp, device=w.device, dtype=torch.bfloat16)
    p = torch.zeros(co, 4, 4, cin_pad, device=w.device, dtype=w.dtype)
    p[..., :ci] = w.permute(0, 2, 3, 1)
    out[:, :16 * cin_pad] = p.reshape(co, 16 * cin_pad)
    return out, kp


def pack_dgrad(w, stride):
    """The dgrad packs of W [Co, Ci, 4, 4]: stride 1, bf16 [Ci, 16 Co] with column (ky * 4 + kx) * Co + co =
    W[co, ci, 3 - ky, 3 - kx]; stride 2, bf16 [4, Ci, 4 Co], class 2 py + px, column (ty * 2 + tx) * Co + co =
    W[co, ci, 3 - py - 2 ty, 3 - px - 2 tx].  Returns (pack, k_pitch)."""
    co, ci = w.shape[:2]
    if stride == 1:
        return w.flip(2, 3).permute(1, 2, 3, 0).reshape(ci, 16 * co).to(torch.bfloat16).contiguous(), 16 * co
    packs = []
    for py in range(2):
        for px in range(2):
            sub = w[:, :, [3 - py, 1 - py]][:, :, :, [3 - px, 1 - px]]
            packs.append(sub.permute(1, 2, 3, 0).reshape(ci, 4 * co))
    return torch.stack(packs).to(torch.bfloat16).contiguous(), 4 * co


class NLayerDiscriminator(nn.Module):
    """nsr.losses.disc.NLayerDiscriminator(input_nc=3, ndf=64, n_layers=3, use_actnorm=False) on libga_b200.so.
    forward(input [N, 3, H, W] CUDA fp32 or bf16) -> fp32 logits [N, 1, Ho, Wo].  Training mode normalises with the
    batch statistics and updates the running ones (momentum 0.1, unbiased variance) whatever the grad mode; eval mode
    uses the running statistics.  Autocast is ignored."""

    def __init__(self, input_nc=3, ndf=64, n_layers=3, use_actnorm=False):
        super().__init__()
        if use_actnorm:
            raise NotImplementedError("NLayerDiscriminator: use_actnorm=True is not built (only BatchNorm2d)")
        if (input_nc, ndf, n_layers) != (INPUT_NC, NDF, N_LAYERS):
            raise NotImplementedError("NLayerDiscriminator: only input_nc=3, ndf=64, n_layers=3 is built, got %s"
                                      % ((input_nc, ndf, n_layers),))
        c = CHANNELS
        self.main = nn.Sequential(
            nn.Conv2d(c[0], c[1], 4, 2, 1), nn.LeakyReLU(SLOPE, True),
            nn.Conv2d(c[1], c[2], 4, 2, 1, bias=False), nn.BatchNorm2d(c[2]), nn.LeakyReLU(SLOPE, True),
            nn.Conv2d(c[2], c[3], 4, 2, 1, bias=False), nn.BatchNorm2d(c[3]), nn.LeakyReLU(SLOPE, True),
            nn.Conv2d(c[3], c[4], 4, 1, 1, bias=False), nn.BatchNorm2d(c[4]), nn.LeakyReLU(SLOPE, True),
            nn.Conv2d(c[4], c[5], 4, 1, 1))

    def _convs(self):
        return [self.main[i] for i in (0, 2, 5, 8, 11)]

    def _bns(self):
        return [self.main[i] for i in (3, 6, 9)]

    def _params(self):
        cv, bn = self._convs(), self._bns()
        return [cv[0].weight, cv[0].bias, cv[1].weight, bn[0].weight, bn[0].bias, cv[2].weight, bn[1].weight,
                bn[1].bias, cv[3].weight, bn[2].weight, bn[2].bias, cv[4].weight, cv[4].bias]

    def forward(self, input):
        x = input
        if x.dim() != 4 or x.shape[1] != INPUT_NC:
            raise ValueError("NLayerDiscriminator: expected images [N, 3, H, W], got %s" % (tuple(x.shape),))
        N, _, H, W = x.shape
        sz = sizes(H, W)
        if N == 0 or sz[-1][0] <= 0 or sz[-1][1] <= 0:
            raise ValueError("NLayerDiscriminator: input %s is too small for a non-empty output (at least 24 x 24)"
                             % (tuple(x.shape),))
        if self.training:
            for k in range(3):
                if N * sz[k + 2][0] * sz[k + 2][1] < 2:
                    raise ValueError("NLayerDiscriminator: BatchNorm %d would see one value per channel in training "
                                     "(input %s)" % (k + 1, tuple(x.shape)))
        if self.training and any(bn.momentum is None for bn in self._bns()):
            raise NotImplementedError("NLayerDiscriminator: BatchNorm momentum=None (a cumulative average) is not "
                                      "built; the reference uses 0.1")
        if not x.is_cuda:
            raise RuntimeError("NLayerDiscriminator runs on CUDA tensors (there is no CPU fallback)")
        if x.dtype not in (torch.float32, torch.bfloat16):
            raise TypeError("NLayerDiscriminator: input must be fp32 or bf16, got %s" % x.dtype)
        params = self._params()
        for p in params + [b for bn in self._bns() for b in (bn.running_mean, bn.running_var)]:
            if p.dtype != torch.float32 or p.device != x.device:
                raise RuntimeError("NLayerDiscriminator: parameters and buffers must be fp32 on the input's device "
                                   "(%s), got %s on %s" % (x.device, p.dtype, p.device))
        return _DiscFn.apply(self, x, *params)


def _ws(n, dev, dtype=torch.float32):
    return torch.empty(n, device=dev, dtype=dtype)


def _forward(mod, x, params):
    """The forward's launches; returns the logits and what the backward needs."""
    L = _lib.lib()
    dev = x.device
    st = _launch.stream(dev)
    N, _, H, W = x.shape
    sz = sizes(H, W)
    training = mod.training
    w1, b1, w2, g2, be2, w3, g3, be3, w4, g4, be4, w5, b5 = [p.detach() for p in params]
    xf = x.detach().to(torch.float32).contiguous()
    xp = torch.empty(N, H, W, 8, device=dev, dtype=torch.bfloat16)
    _lib.check(L.ga_vae_enc_input(_p(xf), N, 3, H, W, 8, _p(xp), 0, 0, 0, None, st), "ga_vae_enc_input")
    w1p, kp1 = pack_forward(w1, 8)
    h1, wd1 = sz[1]
    a1 = torch.empty(N, h1, wd1, 64, device=dev, dtype=torch.bfloat16)
    _lib.check(L.ga_conv4x4_lrelu_bf16(_p(xp), N, H, W, 8, _p(w1p), kp1, _p(b1.contiguous()), 64, 2, _p(a1), st),
               "ga_conv4x4_lrelu_bf16")
    acts, zs, stats = [a1], [], []
    for k, (w, gam, bet, bn) in enumerate(((w2, g2, be2, mod._bns()[0]), (w3, g3, be3, mod._bns()[1]),
                                           (w4, g4, be4, mod._bns()[2]))):
        cin, cout, s = CHANNELS[k + 1], CHANNELS[k + 2], STRIDES[k + 1]
        (hi, wi), (ho, wo) = sz[k + 1], sz[k + 2]
        M = N * ho * wo
        wp, kp = pack_forward(w, cin)
        z = torch.empty(M, cout, device=dev)
        part = torch.empty(-(-M // 128), cout, 2, device=dev) if training else None
        _lib.check(L.ga_conv4x4_stats(_p(acts[-1]), N, hi, wi, cin, _p(wp), kp, cout, s, _p(z), _p(part), st),
                   "ga_conv4x4_stats")
        mean, rstd = _ws(cout, dev), _ws(cout, dev)
        a = torch.empty(N, ho, wo, cout, device=dev, dtype=torch.bfloat16)
        momentum = bn.momentum if training else 0.0
        _lib.check(L.ga_disc_bn_forward(_p(z), _p(part), M, cout, _p(gam), _p(bet), int(training), float(momentum),
                                        float(bn.eps), _p(bn.running_mean), _p(bn.running_var), _p(mean), _p(rstd),
                                        _p(a), st), "ga_disc_bn_forward")
        if training:
            bn.num_batches_tracked.add_(1)
        acts.append(a)
        zs.append(z)
        stats.append((mean, rstd))
    h4, w4s = sz[4]
    h5, w5s = sz[5]
    w5p = w5[0].permute(1, 2, 0).reshape(16, 512).contiguous()
    logits = torch.empty(N, 1, h5, w5s, device=dev)
    _lib.check(L.ga_disc_conv5(_p(acts[3]), N, h4, w4s, _p(w5p), _p(b5.contiguous()), _p(logits), st), "ga_disc_conv5")
    saved = dict(xp=xp, acts=acts, zs=zs, stats=stats, sz=sz, N=N, training=training, w5p=w5p)
    return logits, saved


def _backward(saved, params, g, need):
    """need[0]: the input; need[1:]: the 13 parameters in _params order.  Returns their gradients (None where not
    needed)."""
    L = _lib.lib()
    dev = g.device
    st = _launch.stream(dev)
    N, sz, training = saved["N"], saved["sz"], int(saved["training"])
    acts, zs, stats = saved["acts"], saved["zs"], saved["stats"]
    w1, b1, w2, g2, be2, w3, g3, be3, w4, g4, be4, w5, b5 = [p.detach() for p in params]
    need_x, nw1, nb1, nw2, ng2, nbe2, nw3, ng3, nbe3, nw4, ng4, nbe4, nw5, nb5 = need
    out = [None] * 14
    g5 = g.to(torch.float32).contiguous()
    h4, w4s = sz[4]
    h5, w5s = sz[5]
    M4 = N * h4 * w4s
    # conv 5 -> gy4, BN 4's partials, dW5
    nb = L.ga_disc_conv5_partials(N, h4, w4s)
    gy = torch.empty(M4, 512, device=dev)
    part = torch.empty(nb, 512, 2, device=dev)
    dwp = torch.empty(nb, 16, 512, device=dev) if nw5 else None
    dw5 = torch.empty(16, 512, device=dev) if nw5 else None
    _lib.check(L.ga_disc_conv5_backward(_p(g5), N, h4, w4s, _p(saved["w5p"]), _p(acts[3]), _p(zs[2]),
                                        _p(stats[2][0]), _p(stats[2][1]), _p(gy), _p(part), _p(dwp), _p(dw5), st),
               "ga_disc_conv5_backward")
    if nw5:
        out[12] = dw5.reshape(4, 4, 512).permute(2, 0, 1).unsqueeze(0).contiguous()
    if nb5:
        out[13] = _colsum(L, g5, False, g5.numel(), 1, dev, st)
    convw = (w2, w3, w4)
    gammas = (g2, g3, g4)
    nwk, ngk, nbk = (nw2, nw3, nw4), (ng2, ng3, ng4), (nbe2, nbe3, nbe4)
    slot_w, slot_g, slot_b = (3, 6, 9), (4, 7, 10), (5, 8, 11)
    n_part = nb
    for k in (2, 1, 0):                                   # BatchNorm k + 1, then conv k + 2 (0-based convs k + 1)
        # the gradient at the conv's input, when anything below needs it
        below = need_x or nw1 or nb1 or any(nwk[:k]) or any(ngk[:k]) or any(nbk[:k])
        if not (below or nwk[k] or ngk[k] or nbk[k]):
            break
        cout = CHANNELS[k + 2]
        ho, wo = sz[k + 2]
        M = N * ho * wo
        mean, rstd = stats[k]
        dg = torch.empty(cout, device=dev) if ngk[k] else None
        db = torch.empty(cout, device=dev) if nbk[k] else None
        dz = torch.empty(N, ho, wo, cout, device=dev, dtype=torch.bfloat16)
        kk = torch.empty(cout, 2, device=dev)
        _lib.check(L.ga_disc_bn_backward(_p(gy), _p(zs[k]), M, cout, _p(mean), _p(rstd), _p(gammas[k]), _p(part),
                                         n_part, training, _p(dg), _p(db), _p(kk), _p(dz), st), "ga_disc_bn_backward")
        out[slot_g[k]], out[slot_b[k]] = dg, db
        cin, s = CHANNELS[k + 1], STRIDES[k + 1]
        hi, wi = sz[k + 1]
        if nwk[k]:
            out[slot_w[k]] = _wgrad(L, dz, acts[k], N, hi, wi, cin, cout, s, cin, dev, st)
        if not below:
            break
        wf, kpf = pack_dgrad(convw[k], s)
        if k > 0:
            n_part = L.ga_disc_dgrad_partials(N, hi, wi, s)
            gy = torch.empty(N * hi * wi, cin, device=dev)
            part = torch.empty(n_part, cin, 2, device=dev)
            _lib.check(L.ga_disc_dgrad(_p(dz), N, hi, wi, cout, _p(wf), kpf, cin, s, _p(acts[k]), _p(zs[k - 1]),
                                       _p(stats[k - 1][0]), _p(stats[k - 1][1]), _p(gy), _p(part), None, st),
                       "ga_disc_dgrad")
        else:
            dz1 = torch.empty(N, hi, wi, cin, device=dev, dtype=torch.bfloat16)
            _lib.check(L.ga_disc_dgrad(_p(dz), N, hi, wi, cout, _p(wf), kpf, cin, s, _p(acts[0]), None, None, None,
                                       None, None, _p(dz1), st), "ga_disc_dgrad")
            H, W = sz[0]
            if nw1:
                out[1] = _wgrad(L, dz1, saved["xp"], N, H, W, 8, 64, 2, 3, dev, st)
            if nb1:
                out[2] = _colsum(L, dz1, True, N * hi * wi, 64, dev, st)
            if need_x:
                w1f = w1.to(torch.bfloat16).float().permute(2, 3, 0, 1).reshape(16, 64, 3).contiguous()
                dx = torch.empty(N, 3, H, W, device=dev)
                _lib.check(L.ga_disc_input_backward(_p(dz1), N, H, W, _p(w1f), _p(dx), st), "ga_disc_input_backward")
                out[0] = dx
    return out


def _wgrad(L, dy, x, N, H, W, cin, cout, stride, cin_out, dev, st):
    ho, wo = out_size(H, stride), out_size(W, stride)
    ws = torch.empty(L.ga_disc_wgrad_workspace_bytes(N, ho, wo, cout, cin), device=dev, dtype=torch.uint8)
    dw = torch.empty(cout, cin_out, 4, 4, device=dev)
    _lib.check(L.ga_disc_wgrad(_p(dy), _p(x), N, H, W, cin, cout, stride, cin_out, _p(ws), ws.numel(), _p(dw), st),
               "ga_disc_wgrad")
    return dw


def _colsum(L, x, is_bf16, rows, C, dev, st):
    scratch = torch.empty(L.ga_disc_colsum_scratch_bytes(rows, C), device=dev, dtype=torch.uint8)
    out = torch.empty(C, device=dev)
    _lib.check(L.ga_disc_colsum(_p(x), int(is_bf16), rows, C, _p(scratch), scratch.numel(), _p(out), st),
               "ga_disc_colsum")
    return out


class _DiscFn(torch.autograd.Function):
    """Logits of the discriminator `mod` for input x; the parameters are inputs so autograd routes their gradients
    (accumulated into .grad as for any leaf).  The saved activations belong to this call."""

    @staticmethod
    def forward(ctx, mod, x, *params):
        with torch.cuda.device(x.device), torch.autocast("cuda", enabled=False):
            logits, saved = _forward(mod, x, params)
        # the parameters go through save_for_backward, so an in-place change before backward raises
        ctx.save_for_backward(*params)
        ctx.saved, ctx.x_dtype = saved, x.dtype
        return logits

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        if ctx.saved is None:
            raise RuntimeError("NLayerDiscriminator: the activations of this call were freed by its first backward; "
                               "a second backward through the same call (retain_graph=True) is not supported -- "
                               "call the discriminator again")
        params = ctx.saved_tensors
        need = list(ctx.needs_input_grad[1:])
        with torch.cuda.device(g.device):
            grads = _backward(ctx.saved, params, g, need)
        if grads[0] is not None:
            grads[0] = grads[0].to(ctx.x_dtype)
        grads = [gr if n else None for gr, n in zip(grads, need)]
        ctx.saved = None
        return (None, *grads)
