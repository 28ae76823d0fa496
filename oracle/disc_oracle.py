"""numpy restatement of the PatchGAN discriminator (nsr/losses/disc.py NLayerDiscriminator(3, 64, 3), the library's
gaussiananything_b200.disc): forward in training and eval mode with the running-statistic update, the input and
parameter gradients, and the stride-2 dgrad's parity decomposition.

Exact mode: everything in fp64.  emulate=True: the roundings of include/ga_b200.h Part 11 -- the input, the
convolution weights of convs 1-4, the activations a1..a4 and the gradients dz1..dz4 rounded to bf16, the
pre-normalisation outputs z2..z4, the gradients gy2..gy4 and the logits to fp32 -- with every sum in fp64.

State dicts are {key: array} in the reference's layout (numpy or CPU torch tensors)."""
import numpy as np

STRIDES = (2, 2, 2, 1, 1)
CONVS = ("main.0", "main.2", "main.5", "main.8", "main.11")
BNS = ("main.3", "main.6", "main.9")
SLOPE = 0.2
EPS = 1e-5
MOMENTUM = 0.1


def bf16(a):
    """Round to bf16 (nearest, ties to even), returned as fp64."""
    f = np.ascontiguousarray(a, dtype=np.float32)
    u = f.view(np.uint32).astype(np.uint64)
    u = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return u.astype(np.uint32).view(np.float32).astype(np.float64)


def f32(a):
    return np.asarray(a, dtype=np.float32).astype(np.float64)


def _np(sd):
    return {k: np.asarray(v.detach().cpu().numpy() if hasattr(v, "detach") else v, dtype=np.float64)
            for k, v in sd.items()}


def out_size(h, s):
    return (h - 2) // s + 1


def conv(x, w, s, b=None):
    """4x4 pad-1 convolution, x [N, Ci, H, W], w [Co, Ci, 4, 4] -> [N, Co, Ho, Wo], fp64."""
    N, _, H, W = x.shape
    Ho, Wo = out_size(H, s), out_size(W, s)
    xp = np.pad(x, ((0, 0), (0, 0), (1, 1), (1, 1)))
    out = np.zeros((w.shape[0], N, Ho, Wo))
    for ky in range(4):
        for kx in range(4):
            xs = xp[:, :, ky:ky + s * (Ho - 1) + 1:s, kx:kx + s * (Wo - 1) + 1:s]
            out += np.tensordot(w[:, :, ky, kx], xs, axes=([1], [1]))
    out = out.transpose(1, 0, 2, 3)
    return out if b is None else out + b.reshape(1, -1, 1, 1)


def conv_dgrad(g, w, s, H, W):
    """d(sum g * conv(x)) / dx for x of [N, Ci, H, W]: the scatter of every tap, fp64."""
    N, _, Ho, Wo = g.shape
    dxp = np.zeros((N, w.shape[1], H + 2, W + 2))
    for ky in range(4):
        for kx in range(4):
            t = np.tensordot(g, w[:, :, ky, kx], axes=([1], [0])).transpose(0, 3, 1, 2)
            dxp[:, :, ky:ky + s * (Ho - 1) + 1:s, kx:kx + s * (Wo - 1) + 1:s] += t
    return dxp[:, :, 1:H + 1, 1:W + 1]


def conv_dgrad_parity(g, w, H, W):
    """The stride-2 dgrad as include/ga_b200.h Part 11 decomposes it: input pixel (2a + py, 2b + px) gets the 2x2
    stride-1 convolution of g at rows a - 1 + py + ty, columns b - 1 + px + tx with W[:, :, 3 - py - 2 ty,
    3 - px - 2 tx]."""
    N, _, Ho, Wo = g.shape
    dx = np.zeros((N, w.shape[1], H, W))
    gp = np.pad(g, ((0, 0), (0, 0), (1, 1), (1, 1)))
    for py in range(2):
        for px in range(2):
            Ha, Wa = (H - py + 1) // 2, (W - px + 1) // 2
            acc = np.zeros((N, w.shape[1], Ha, Wa))
            for ty in range(2):
                for tx in range(2):
                    r0, c0 = py + ty, px + tx                 # row a - 1 + py + ty of g is row a + py + ty of gp
                    gs = gp[:, :, r0:r0 + Ha, c0:c0 + Wa]
                    if gs.shape[2] < Ha or gs.shape[3] < Wa:
                        gs = np.pad(gs, ((0, 0), (0, 0), (0, Ha - gs.shape[2]), (0, Wa - gs.shape[3])))
                    acc += np.tensordot(gs, w[:, :, 3 - py - 2 * ty, 3 - px - 2 * tx], axes=([1], [0])).transpose(0, 3, 1, 2)
            dx[:, :, py::2, px::2] = acc
    return dx


def conv_wgrad(g, x, s):
    """d(sum g * conv(x)) / dW [Co, Ci, 4, 4], fp64."""
    _, _, Ho, Wo = g.shape
    xp = np.pad(x, ((0, 0), (0, 0), (1, 1), (1, 1)))
    dw = np.zeros((g.shape[1], x.shape[1], 4, 4))
    for ky in range(4):
        for kx in range(4):
            xs = xp[:, :, ky:ky + s * (Ho - 1) + 1:s, kx:kx + s * (Wo - 1) + 1:s]
            dw[:, :, ky, kx] = np.tensordot(g, xs, axes=([0, 2, 3], [0, 2, 3]))
    return dw


def lrelu(v):
    return np.where(v > 0, v, SLOPE * v)


def forward(sd, x, training=True, emulate=False):
    """Logits [N, 1, Ho, Wo] and the cache for backward(); in training mode also the updated running statistics
    {key: array} (the state dict is not modified)."""
    p = _np(sd)
    rb = bf16 if emulate else (lambda a: a)
    r32 = f32 if emulate else (lambda a: a)
    x = np.asarray(x, dtype=np.float64)
    cache = {"x": rb(x), "training": training, "acts": [], "zs": [], "stats": [], "emulate": emulate, "p": p}
    a = rb(lrelu(conv(cache["x"], rb(p["main.0.weight"]), 2, p["main.0.bias"])))
    cache["acts"].append(a)
    new = {}
    for k in range(3):
        w = rb(p[CONVS[k + 1] + ".weight"])
        z = r32(conv(a, w, STRIDES[k + 1]))
        bn = BNS[k]
        if training:
            mean = z.mean(axis=(0, 2, 3))
            var = z.var(axis=(0, 2, 3))
            M = z.shape[0] * z.shape[2] * z.shape[3]
            new[bn + ".running_mean"] = (1 - MOMENTUM) * p[bn + ".running_mean"] + MOMENTUM * mean
            new[bn + ".running_var"] = (1 - MOMENTUM) * p[bn + ".running_var"] + MOMENTUM * var * M / (M - 1)
            new[bn + ".num_batches_tracked"] = p[bn + ".num_batches_tracked"] + 1
        else:
            mean, var = p[bn + ".running_mean"], p[bn + ".running_var"]
        rstd = 1.0 / np.sqrt(var + EPS)
        if emulate:
            mean, rstd = f32(mean), f32(rstd)
        xhat = (z - mean.reshape(1, -1, 1, 1)) * rstd.reshape(1, -1, 1, 1)
        y = xhat * p[bn + ".weight"].reshape(1, -1, 1, 1) + p[bn + ".bias"].reshape(1, -1, 1, 1)
        a = rb(lrelu(y))
        cache["acts"].append(a)
        cache["zs"].append(z)
        cache["stats"].append((mean, rstd, xhat))
    logits = r32(conv(a, p["main.11.weight"], 1, p["main.11.bias"]))
    return logits, cache, new


def backward(cache, g):
    """Gradients of sum(g * logits): (dx, {param key: gradient})."""
    p, emulate = cache["p"], cache["emulate"]
    rb = bf16 if emulate else (lambda a: a)
    r32 = f32 if emulate else (lambda a: a)
    acts, zs, stats = cache["acts"], cache["zs"], cache["stats"]
    g = np.asarray(g, dtype=np.float64)
    grads = {"main.11.weight": conv_wgrad(g, acts[3], 1), "main.11.bias": g.sum(axis=(0, 2, 3))}
    up = conv_dgrad(g, p["main.11.weight"], 1, *acts[3].shape[2:])
    for k in (2, 1, 0):
        bn = BNS[k]
        gy = r32(np.where(acts[k + 1] > 0, up, SLOPE * up))
        mean, rstd, xhat = stats[k]
        grads[bn + ".bias"] = gy.sum(axis=(0, 2, 3))
        grads[bn + ".weight"] = (gy * xhat).sum(axis=(0, 2, 3))
        gam = p[bn + ".weight"].reshape(1, -1, 1, 1) * rstd.reshape(1, -1, 1, 1)
        if cache["training"]:
            M = gy.shape[0] * gy.shape[2] * gy.shape[3]
            k1 = (grads[bn + ".bias"] / M).reshape(1, -1, 1, 1)
            k2 = (grads[bn + ".weight"] / M).reshape(1, -1, 1, 1)
            dz = rb(gam * (gy - k1 - xhat * k2))
        else:
            dz = rb(gam * gy)
        w = rb(p[CONVS[k + 1] + ".weight"])
        grads[CONVS[k + 1] + ".weight"] = conv_wgrad(dz, acts[k], STRIDES[k + 1])
        up = conv_dgrad(dz, w, STRIDES[k + 1], *acts[k].shape[2:])
    dz1 = rb(np.where(acts[0] > 0, up, SLOPE * up))
    w1 = rb(p["main.0.weight"])
    grads["main.0.weight"] = conv_wgrad(dz1, cache["x"], 2)
    grads["main.0.bias"] = dz1.sum(axis=(0, 2, 3))
    dx = conv_dgrad(dz1, w1, 2, *cache["x"].shape[2:])
    return dx, grads


def hinge_d_loss(lr, lf):
    """0.5 (mean(relu(1 - logits_real)) + mean(relu(1 + logits_fake))), and its gradients to the two logits."""
    loss = 0.5 * (np.maximum(1 - lr, 0).mean() + np.maximum(1 + lf, 0).mean())
    gr = np.where(1 - lr > 0, -0.5 / lr.size, 0.0)
    gf = np.where(1 + lf > 0, 0.5 / lf.size, 0.0)
    return loss, gr, gf


def d_step_grads(sd, real, fake, emulate=False):
    """The reference's d-step on one state: train-mode logits of the real batch, then of the fake batch (two BatchNorm
    batches), hinge_d_loss and its parameter gradients summed over both calls; the running statistics after both."""
    lr, cr, new_r = forward(sd, real, True, emulate)
    sd2 = dict(_np(sd))
    sd2.update(new_r)
    lf, cf, new_f = forward(sd2, fake, True, emulate)
    loss, gr, gf = hinge_d_loss(lr, lf)
    _, g_r = backward(cr, gr)
    _, g_f = backward(cf, gf)
    grads = {k: g_r[k] + g_f[k] for k in g_r}
    sd2.update(new_f)
    return dict(lr=lr, lf=lf, loss=loss, grads=grads, state=sd2, cache_fake=cf)
