"""Image-quality metrics on the library's kernels: LPIPS with the VGG16 backbone and SSIM (include/ga_b200.h Part 8).

  LPIPS   mirrors lpips.LPIPS(net="vgg", version="0.1", spatial=False), the perceptual metric of the reference's VAE
          objective (nsr/losses/builder.py LPIPSLoss; the same network and formulas as
          sgm/modules/autoencoding/lpips/loss/lpips.py): ScalingLayer, VGG16 `features` cut at relu1_2 .. relu5_3,
          unit-normalised features (eps 1e-10), squared difference, a bias-free 1x1 NetLinLayer per tap, spatial mean,
          sum over the five taps.
  LPIPSLoss  mirrors LPIPSLoss of nsr/losses/builder.py: loss_weight * LPIPS(target, pred).mean(), differentiable
          in pred and / or target through the Part 9 backward (input gradients only; the network is frozen).
  ssim    _ssim of nsr/losses/builder.py with create_window(11, 3) and size_average=False: per-image SSIM.

Precision: the 13 convolutions take bf16 operands and keep bf16 ReLU outputs (fp32 accumulation), as every network
here; the head and the reductions run in fp32.  Rounding noise enters LPIPS squared, so the bf16 error is a small
positive bias (INTEGRATION.md section 3g).  The backward keeps bf16 gradients between the convolutions, fp32 at the
pooled maps, the head and the input (INTEGRATION.md section 3h).

Weights are never downloaded: state_dict= (the LPIPS module layout), or vgg_path= / lin_path=, or the default local
files torch.hub.get_dir()/checkpoints/vgg16-397923af.pth (torchvision's VGG16) and .../checkpoints/vgg.pth (the
LPIPS linear layers, `lin{k}.model.1.weight`).
"""
import math
import os

import torch

from . import _launch, _lib
from ._launch import ptr as _p

TAPS = 5
CHNS = (64, 128, 256, 512, 512)
# VGG16 `features` index of each 3x3 convolution, by slice of the LPIPS network (slice k ends at tap k's ReLU)
SLICES = ((0, 2), (5, 7), (10, 12, 14), (17, 19, 21), (24, 26, 28))
SHIFT = (-0.030, -0.088, -0.188)
SCALE = (0.458, 0.448, 0.450)
HEAD_BLOCKS = 128                          # GA_LPIPS_HEAD_BLOCKS of include/ga_b200.h
SSIM_WINDOW = 11                           # GA_SSIM_WINDOW
VGG_FILE = "vgg16-397923af.pth"            # torchvision's VGG16 checkpoint
LIN_FILE = "vgg.pth"                       # the LPIPS package's linear layers for net="vgg", version 0.1
MIN_SIZE = 16                              # relu5_3 is (H >> 4) x (W >> 4)


def _conv_list():
    """[(slice k, features index i, Cin, Cout)] of the 13 convolutions in order."""
    out, cin = [], 3
    for k, idx in enumerate(SLICES):
        for i in idx:
            out.append((k, i, cin, CHNS[k]))
            cin = CHNS[k]
    return out


CONVS = _conv_list()


def state_dict_shapes():
    """{key: shape} of the LPIPS module's state dict (tests/golden/lpips_vgg_keys.json): scaling_layer.shift / scale
    [1, 3, 1, 1], net.slice{k}.{i}.weight [Cout, Cin, 3, 3] / .bias [Cout], lin{k}.model.1.weight [1, C, 1, 1]."""
    s = {"scaling_layer.shift": (1, 3, 1, 1), "scaling_layer.scale": (1, 3, 1, 1)}
    for k, i, cin, cout in CONVS:
        s["net.slice%d.%d.weight" % (k + 1, i)] = (cout, cin, 3, 3)
        s["net.slice%d.%d.bias" % (k + 1, i)] = (cout,)
    for k, c in enumerate(CHNS):
        s["lin%d.model.1.weight" % k] = (1, c, 1, 1)
    return s


OPTIONAL_KEYS = ("scaling_layer.shift", "scaling_layer.scale")


def check_state_dict(sd):
    """Strict: every key of the layout is present with its shape (the scaling-layer buffers may be absent), and no
    other key.  Raises RuntimeError naming the missing, unexpected or misshapen keys."""
    want = state_dict_shapes()
    missing = [k for k in want if k not in sd and k not in OPTIONAL_KEYS]
    unexpected = [k for k in sd if k not in want]
    if missing or unexpected:
        raise RuntimeError("LPIPS state dict does not match the VGG layout: missing keys %s, unexpected keys %s"
                           % (missing, unexpected))
    bad = ["%s %s (expected %s)" % (k, tuple(sd[k].shape), want[k]) for k in sd if tuple(sd[k].shape) != want[k]]
    if bad:
        raise RuntimeError("LPIPS state dict: wrong shapes: %s" % ", ".join(bad))


def default_paths():
    d = os.path.join(torch.hub.get_dir(), "checkpoints")
    return os.path.join(d, VGG_FILE), os.path.join(d, LIN_FILE)


def state_dict_from_files(vgg_path=None, lin_path=None):
    """The LPIPS module layout from torchvision's VGG16 checkpoint (features.{i}.weight / bias of the 13 convolutions;
    classifier.* is ignored) and the LPIPS linear-layer file (lin{k}.model.1.weight).  Local files only; a missing
    file raises RuntimeError saying where it goes."""
    dv, dl = default_paths()
    vgg_path, lin_path = vgg_path or dv, lin_path or dl
    for what, path, name in (("VGG16", vgg_path, VGG_FILE), ("LPIPS linear-layer", lin_path, LIN_FILE)):
        if not os.path.exists(path):
            raise RuntimeError("LPIPS weights not found: pass state_dict=, or place the %s file %s at %s "
                               "(nothing is downloaded)" % (what, name, path))
    vgg = torch.load(vgg_path, map_location="cpu", weights_only=True)
    lin = torch.load(lin_path, map_location="cpu", weights_only=True)
    sd = {}
    for k, i, _, _ in CONVS:
        for p in ("weight", "bias"):
            src = "features.%d.%s" % (i, p)
            if src not in vgg:
                raise RuntimeError("VGG16 checkpoint %s lacks %s" % (vgg_path, src))
            sd["net.slice%d.%d.%s" % (k + 1, i, p)] = vgg[src]
    for k in range(TAPS):
        src = "lin%d.model.1.weight" % k
        if src not in lin:
            raise RuntimeError("LPIPS linear-layer file %s lacks %s" % (lin_path, src))
        sd[src] = lin[src]
    return sd


def gaussian_window(window_size=SSIM_WINDOW, sigma=1.5):
    """create_window(window_size, .)[0, 0] as the reference computes it: the 1D Gaussian in fp32, normalised by its
    fp32 sum, and its fp32 outer product."""
    g = torch.tensor([math.exp(-(x - window_size // 2) ** 2 / float(2 * sigma ** 2)) for x in range(window_size)],
                     dtype=torch.float32)
    g = (g / g.sum()).unsqueeze(1)
    return g.mm(g.t()).float()


def _check_pair(in0, in1, what, min_size=1, allow_grad=False):
    if in0.dim() != 4 or in0.shape[1] != 3:
        raise ValueError("%s: expected images [N, 3, H, W], got %s" % (what, tuple(in0.shape)))
    if tuple(in0.shape) != tuple(in1.shape):
        raise ValueError("%s: the two inputs differ in shape: %s and %s" % (what, tuple(in0.shape), tuple(in1.shape)))
    if in0.shape[0] == 0 or in0.shape[2] < min_size or in0.shape[3] < min_size:
        raise ValueError("%s: N must be positive and H, W at least %d, got %s" % (what, min_size, tuple(in0.shape)))
    if not (in0.is_cuda and in1.is_cuda):
        raise RuntimeError("%s runs on CUDA tensors (there is no CPU fallback)" % what)
    if not allow_grad and torch.is_grad_enabled() and (in0.requires_grad or in1.requires_grad):
        raise RuntimeError("%s is inference-only (no autograd through the CUDA kernels): call it under torch.no_grad() "
                           "or on detached inputs" % what)


def ssim(img1, img2, window_size=SSIM_WINDOW):
    """Per-image SSIM [N] (fp32) of img1, img2 [N, 3, H, W] in [0, 1]: _ssim(..., size_average=False) with the
    reference's 11 x 11 Gaussian window (sigma 1.5) and zero padding."""
    if window_size != SSIM_WINDOW:
        raise NotImplementedError("ssim: only window_size=%d is built" % SSIM_WINDOW)
    _check_pair(img1, img2, "ssim")
    N, _, H, W = img1.shape
    dev = img1.device
    L = _lib.lib()
    with torch.cuda.device(dev), torch.no_grad():
        a = img1.to(dtype=torch.float32).contiguous()
        b = img2.to(device=dev, dtype=torch.float32).contiguous()
        win = gaussian_window(window_size).to(dev)
        scratch = torch.empty(L.ga_ssim_scratch_bytes(N, H, W), dtype=torch.uint8, device=dev)
        out = torch.empty(N, device=dev)
        _lib.check(L.ga_ssim(_p(a), _p(b), N, H, W, _p(win), _p(scratch), scratch.numel(), _p(out),
                             _launch.stream(dev)), "ga_ssim")
    return out


class LPIPS:
    """lpips.LPIPS(net="vgg", version="0.1", spatial=False) on libga_b200.so.  `forward(in0, in1)` (or calling the
    object) returns [N, 1, 1, 1] fp32, and with retPerLayer=True also the five per-tap values [N, 1, 1, 1].

    Pairs go through the network `chunk` at a time, so activation memory stays bounded (the first two layers'
    outputs for 8 pairs at 512^2 take 1.07 GB); every kernel works per image or per pair, so the result has the same
    bits whatever the chunking.  Each (chunk, H, W) launch sequence is captured once into a CUDA graph and replayed;
    `use_graph = False` (or GA_B200_LPIPS_GRAPH=0) launches eagerly with the same bits."""
    use_graph = _launch.graph_switch()
    chunk = 8

    def __init__(self, net="vgg", version="0.1", spatial=False, state_dict=None, vgg_path=None, lin_path=None,
                 device="cuda"):
        if net != "vgg":
            raise NotImplementedError("LPIPS: only net='vgg' is built (AlexNet and SqueezeNet are not)")
        if version != "0.1":
            raise NotImplementedError("LPIPS: only version='0.1' is built")
        if spatial:
            raise NotImplementedError("LPIPS: spatial=True is not built (the spatial mean is fused into the head)")
        sd = state_dict if state_dict is not None else state_dict_from_files(vgg_path, lin_path)
        check_state_dict(sd)
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("gaussiananything_b200 LPIPS needs a CUDA device (no CPU fallback)")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.L = _lib.lib()
        dev = self.device
        f32 = lambda t: t.detach().to(device=dev, dtype=torch.float32).contiguous()
        self.shift = f32(sd.get("scaling_layer.shift", torch.tensor(SHIFT)).reshape(3))
        self.scale = f32(sd.get("scaling_layer.scale", torch.tensor(SCALE)).reshape(3))
        self.convs = []
        for j, (k, i, cin, cout) in enumerate(CONVS):
            w = sd["net.slice%d.%d.weight" % (k + 1, i)].detach().float().cpu()
            cp = _launch.round_up(cin, 8)                   # the packed input has 8 channels, 3 used
            kp = _launch.round_up(9 * cp, 64)
            wp = torch.zeros(cout, 3, 3, cp)
            wp[..., :cin] = w.permute(0, 2, 3, 1)
            packed = torch.zeros(cout, kp)
            packed[:, :9 * cp] = wp.reshape(cout, 9 * cp)
            self.convs.append(dict(tap=k, cin=cp, cout=cout, kp=kp, w=packed.to(device=dev, dtype=torch.bfloat16),
                                   b=f32(sd["net.slice%d.%d.bias" % (k + 1, i)]),
                                   last=j + 1 == len(CONVS) or CONVS[j + 1][0] != k))    # its ReLU is tap k
            if j:                                            # the dgrad's weights (include/ga_b200.h Part 9)
                wf, self.convs[-1]["kpf"] = flip_pack(w)
                self.convs[-1]["wf"] = wf.to(dev)
        # features.0's dgrad in ga_lpips_input_backward: w_flip [9, 64, 3] = W0[co, c, 2 - ky, 2 - kx]
        w0 = sd["net.slice1.0.weight"].detach().float().cpu().to(torch.bfloat16).float()
        self.w0_flip = w0.flip(2, 3).permute(2, 3, 0, 1).reshape(9, CHNS[0], 3).contiguous().to(dev)
        self.lin = [f32(sd["lin%d.model.1.weight" % k].reshape(-1)) for k in range(TAPS)]
        self._graphs = _launch.GraphCache("GA_B200_LPIPS_GRAPH")          # (chunk, H, W) -> graph

    def eval(self):
        return self

    # ---- launches of one chunk of n pairs
    def _network(self, in0, in1, normalize, want_taps=False):
        n, _, H, W = in0.shape
        dev, L = self.device, self.L
        st = _launch.stream(dev)
        x = torch.empty(2 * n, H, W, 8, device=dev, dtype=torch.bfloat16)
        _lib.check(L.ga_lpips_pack(_p(in0), _p(in1), n, H, W, int(bool(normalize)), _p(self.shift), _p(self.scale),
                                   _p(x), st), "ga_lpips_pack")
        partial = torch.empty(TAPS, n, HEAD_BLOCKS, device=dev)
        taps = []
        h, w, tap = H, W, 0
        for cv in self.convs:
            if cv["tap"] != tap:                                           # a 2x2 max pool starts every later slice
                y = torch.empty(2 * n, h // 2, w // 2, x.shape[-1], device=dev, dtype=torch.bfloat16)
                _lib.check(L.ga_maxpool2x2_bf16(_p(x), 2 * n, h, w, x.shape[-1], _p(y), st), "ga_maxpool2x2_bf16")
                x, h, w, tap = y, h // 2, w // 2, cv["tap"]
            y = torch.empty(2 * n, h, w, cv["cout"], device=dev, dtype=torch.bfloat16)
            _lib.check(L.ga_conv3x3_relu_bf16(_p(x), 2 * n, h, w, cv["cin"], _p(cv["w"]), cv["kp"], _p(cv["b"]),
                                              cv["cout"], _p(y), st), "ga_conv3x3_relu_bf16")
            x = y
            if cv["last"]:
                _lib.check(L.ga_lpips_head(_p(x), n, h, w, cv["cout"], _p(self.lin[tap]), _p(partial[tap]), st),
                           "ga_lpips_head")
                if want_taps:
                    taps.append(x)
        out = torch.empty(n, TAPS + 1, device=dev)
        _lib.check(L.ga_lpips_reduce(_p(partial), n, H, W, _p(out), st), "ga_lpips_reduce")
        return {"out": out, "taps": taps} if want_taps else {"out": out}

    def _inputs(self, in0, in1):
        _check_pair(in0, in1, "LPIPS", MIN_SIZE)
        f = lambda t: t.to(device=self.device, dtype=torch.float32).contiguous()
        return f(in0), f(in1)

    def table(self, in0, in1, normalize=False):
        """fp32 [N, 6]: the five per-tap spatial means and their sum (ga_lpips_reduce), pairs `chunk` at a time."""
        a, b = self._inputs(in0, in1)
        N, _, H, W = a.shape
        rows = []
        with torch.cuda.device(self.device), torch.no_grad():
            for s in range(0, N, self.chunk):
                c0, c1 = a[s:s + self.chunk], b[s:s + self.chunk]
                n = c0.shape[0]
                launches = lambda x0, x1: self._network(x0, x1, normalize)
                rows.append(self._graphs.run((n, H, W, bool(normalize)), launches, [c0, c1])["out"])
        return torch.cat(rows, 0)

    def features(self, in0, in1, normalize=False):
        """The five tap activations, bf16 NHWC [2N, h, w, C] (in0's images first), and the [N, 6] table of one eager
        pass over all N pairs (no chunking, no graph): for tests and inspection."""
        a, b = self._inputs(in0, in1)
        with torch.cuda.device(self.device), torch.no_grad():
            r = self._network(a, b, normalize, want_taps=True)
        return r["taps"], r["out"]

    def forward(self, in0, in1, retPerLayer=False, normalize=False):
        t = self.table(in0, in1, normalize)
        val = t[:, TAPS].reshape(-1, 1, 1, 1)
        if retPerLayer:
            return val, [t[:, k].reshape(-1, 1, 1, 1) for k in range(TAPS)]
        return val

    __call__ = forward

    # ---- differentiable values (LPIPSLoss): Part 9
    def values(self, in0, in1, normalize=False):
        """Per-pair LPIPS [N, 1, 1, 1], differentiable in whichever input requires grad (with grad mode on).
        Otherwise it is forward(): the graphs run and nothing is saved."""
        if not (torch.is_grad_enabled() and (in0.requires_grad or in1.requires_grad)):
            return self.forward(in0, in1, normalize=normalize)
        _check_pair(in0, in1, "LPIPS", MIN_SIZE, allow_grad=True)
        sides = tuple(s for s, t in enumerate((in0, in1)) if t.requires_grad)
        f = lambda t: t.to(device=self.device, dtype=torch.float32).contiguous()
        return _LPIPSGrad.apply(self, bool(normalize), sides, f(in0), f(in1)).reshape(-1, 1, 1, 1)

    def _forward_saving(self, in0, in1, normalize, sides):
        """One chunk of n pairs, launched eagerly into fresh tensors that belong to the caller: the [n, 6] table, the
        five taps [2n, h, w, C], and for each side in `sides` its 13 ReLU outputs [n, h, w, C] (the taps as views).
        The two sides run their convolutions apart, so the other side's inner activations are freed as they go; a
        convolution's pixels do not depend on the batch, so the values are forward()'s bits."""
        n, _, H, W = in0.shape
        dev, L = self.device, self.L
        st = _launch.stream(dev)
        x = torch.empty(2 * n, H, W, 8, device=dev, dtype=torch.bfloat16)
        _lib.check(L.ga_lpips_pack(_p(in0), _p(in1), n, H, W, int(bool(normalize)), _p(self.shift), _p(self.scale),
                                   _p(x), st), "ga_lpips_pack")
        partial = torch.empty(TAPS, n, HEAD_BLOCKS, device=dev)
        xs, taps, acts = [x[:n], x[n:]], [], {s: [] for s in sides}
        h, w, tap = H, W, 0
        for cv in self.convs:
            if cv["tap"] != tap:
                y = torch.empty(2 * n, h // 2, w // 2, cv["cin"], device=dev, dtype=torch.bfloat16)
                _lib.check(L.ga_maxpool2x2_bf16(_p(taps[-1]), 2 * n, h, w, cv["cin"], _p(y), st), "ga_maxpool2x2_bf16")
                xs, h, w, tap = [y[:n], y[n:]], h // 2, w // 2, cv["tap"]
            if cv["last"]:
                y = torch.empty(2 * n, h, w, cv["cout"], device=dev, dtype=torch.bfloat16)
                ys = [y[:n], y[n:]]
            else:
                ys = [torch.empty(n, h, w, cv["cout"], device=dev, dtype=torch.bfloat16) for _ in range(2)]
            for s in range(2):
                _lib.check(L.ga_conv3x3_relu_bf16(_p(xs[s]), n, h, w, cv["cin"], _p(cv["w"]), cv["kp"], _p(cv["b"]),
                                                  cv["cout"], _p(ys[s]), st), "ga_conv3x3_relu_bf16")
                if s in acts:
                    acts[s].append(ys[s])
            xs = ys
            if cv["last"]:
                _lib.check(L.ga_lpips_head(_p(y), n, h, w, cv["cout"], _p(self.lin[tap]), _p(partial[tap]), st),
                           "ga_lpips_head")
                taps.append(y)
        out = torch.empty(n, TAPS + 1, device=dev)
        _lib.check(L.ga_lpips_reduce(_p(partial), n, H, W, _p(out), st), "ga_lpips_reduce")
        return {"out": out, "taps": taps, "acts": acts, "n": n, "H": H, "W": W}

    def _backward_side(self, saved, side, g, normalize, dx):
        """d(sum_i g_i LPIPS_i) / d(images of `side`) of one chunk into dx fp32 [n, 3, H, W] (contiguous)."""
        n, H, W = saved["n"], saved["H"], saved["W"]
        acts, taps = saved["acts"][side], saved["taps"]
        dev, L = self.device, self.L
        st = _launch.stream(dev)
        grad, dpool = None, None                 # bf16 at the current conv's pre-activation; fp32 at a pooled map
        for j in range(len(self.convs) - 1, -1, -1):
            cv = self.convs[j]
            k = cv["tap"]
            h, w = H >> k, W >> k
            if cv["last"]:
                grad = torch.empty(n, h, w, cv["cout"], device=dev, dtype=torch.bfloat16)
                _lib.check(L.ga_lpips_tap_backward(_p(taps[k]), n, h, w, cv["cout"], side, _p(self.lin[k]), _p(g),
                                                   _p(dpool), _p(grad), st), "ga_lpips_tap_backward")
            if j == 0:
                _lib.check(L.ga_lpips_input_backward(_p(grad), n, H, W, _p(self.w0_flip), _p(self.scale),
                                                     int(bool(normalize)), _p(dx), st), "ga_lpips_input_backward")
                break
            if self.convs[j - 1]["tap"] == k:    # inside the slice: through the lower conv's ReLU
                out = torch.empty(n, h, w, cv["cin"], device=dev, dtype=torch.bfloat16)
                _lib.check(L.ga_conv3x3_mask_bf16(_p(grad), n, h, w, cv["cout"], _p(cv["wf"]), cv["kpf"], cv["cin"],
                                                  _p(acts[j - 1]), _p(out), st), "ga_conv3x3_mask_bf16")
                grad = out
            else:                                # the slice's first conv: to the pooled map of tap k - 1, fp32
                dpool = torch.empty(n, h, w, cv["cin"], device=dev)
                _lib.check(L.ga_conv3x3_bf16(_p(grad), n, h, w, cv["cout"], _p(cv["wf"]), cv["kpf"], None, cv["cin"],
                                             1, None, _p(dpool), None, st), "ga_conv3x3_bf16")
                grad = None


def flip_pack(w):
    """The dgrad weights of a 3x3 convolution W [Co, Ci, 3, 3] (fp32, CPU): bf16 [Ci, kp] in the packed layout with
    Cout = Ci, Cin = Co, column (ky * 3 + kx) * Co + co = W[co, ci, 2 - ky, 2 - kx]; and kp = 9 Co rounded up to 64."""
    co, ci = w.shape[:2]
    kp = _launch.round_up(9 * co, 64)
    packed = torch.zeros(ci, kp)
    packed[:, :9 * co] = w.flip(2, 3).permute(1, 2, 3, 0).reshape(ci, 9 * co)
    return packed.to(torch.bfloat16), kp


class _LPIPSGrad(torch.autograd.Function):
    """Per-pair LPIPS [N] of fp32 contiguous in0, in1 with the activations saved for `sides`, pairs `chunk` at a
    time; backward runs the Part 9 chain per chunk and side.  The saved tensors belong to this context (allocated per
    call, never a graph's buffers) and are freed with the autograd graph."""

    @staticmethod
    def forward(ctx, model, normalize, sides, in0, in1):
        N = in0.shape[0]
        with torch.cuda.device(model.device):
            chunks = [model._forward_saving(in0[s:s + model.chunk], in1[s:s + model.chunk], normalize, sides)
                      for s in range(0, N, model.chunk)]
        ctx.model, ctx.normalize, ctx.sides, ctx.chunks, ctx.shape = model, normalize, sides, chunks, tuple(in0.shape)
        return torch.cat([c["out"][:, TAPS] for c in chunks])

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gval):
        model, chunks = ctx.model, ctx.chunks
        g = gval.to(device=model.device, dtype=torch.float32).contiguous()
        dx = [torch.empty(ctx.shape, device=model.device) if s in ctx.sides else None for s in range(2)]
        with torch.cuda.device(model.device):
            s0 = 0
            for c in chunks:
                n = c["n"]
                for s in ctx.sides:
                    model._backward_side(c, s, g[s0:s0 + n], ctx.normalize, dx[s][s0:s0 + n])
                s0 += n
        return None, None, None, dx[0], dx[1]


class LPIPSLoss(torch.nn.Module):
    """LPIPSLoss of nsr/losses/builder.py on the library's LPIPS: forward(pred, target) = loss_weight *
    LPIPS(target, pred).mean(), a 0-dim fp32 tensor, differentiable in whichever of pred and target requires grad.
    Inputs may be non-contiguous views (the reference's centre crops) of any float dtype; gradients come back in the
    input's dtype and shape.  `lpips=` takes an existing LPIPS; otherwise one is built from the local weight files
    (raising as LPIPS does when they are absent).  use_input_norm and range_norm are accepted and unused, as in the
    reference; so is conf_sigma_percl."""

    def __init__(self, loss_weight=1.0, use_input_norm=True, range_norm=True, lpips=None):
        super().__init__()
        self.perceptual = lpips if lpips is not None else LPIPS(net="vgg", spatial=False)
        self.loss_weight = loss_weight
        self.use_input_norm = use_input_norm
        self.range_norm = range_norm

    def forward(self, pred, target, conf_sigma_percl=None):
        return self.loss_weight * self.perceptual.values(target, pred).mean()
