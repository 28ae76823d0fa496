"""Writes tests/golden/lpips_small.npz and tests/golden/lpips_vgg_keys.json from the reference's own LPIPS and SSIM.

LPIPS is the reference's sgm/modules/autoencoding/lpips/loss/lpips.py (the VGG network and formulas of
lpips.LPIPS(net="vgg"), which nsr/losses/builder.py uses); SSIM is create_window and _ssim of nsr/losses/builder.py
(imported through _ref_stubs.py, which stands in for the absent kornia, lpips and other third-party modules; the few
others its imports reach, such as torchtyping for annotations, get an empty stub here).  Nothing
is fetched: before any instance is built, torchvision.models.vgg16 is replaced by a constructor with weights=None and
LPIPS.load_from_pretrained by a no-op; `requests` in lpips/util.py is stubbed if it is absent.  The module's
state_dict() keys and shapes go to lpips_vgg_keys.json.

Weights: oracle.lpips_oracle.random_state_dict(SEED) -- Kaiming-normal convolutions with N(0, 0.05) biases (so the
bias path is exercised) and U(0, 0.2) linear layers -- loaded strictly into the reference module.  They are ~59 MB, so
they are not stored: the file keeps per-key sums and first values, and the tests regenerate the weights from the seed
and check those first.  Run in fp32 on the CPU.

Inputs, in [-1, 1]: views 0, 1, 5 of the committed chunk (tests/golden/gbuffer_chunk), area-downsampled to 64 x 64 and
to 50 x 70 (not a multiple of 16), paired with another view, a noisy copy (sigma 0.05), a 3x3 box blur and a 2-pixel
shift.  Stored per size: in0, in1 [N, 3, H, W]; per_tap [N, 5] (the reference's spatial averages, captured from its own
forward) and value [N]; ssim [N] of (in0 + 1) / 2 against (in1 + 1) / 2, run in fp64 on the fp32 window (in fp32,
E[x^2] - mu^2 cancels to errors of ~2e-5 in SSIM, too coarse to check a restatement against).

    python tests/golden/make_lpips_golden.py
"""
import importlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import _ref_stubs  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

SEED = 0
OUT = os.path.join(HERE, "lpips_small.npz")
KEYS = os.path.join(HERE, "lpips_vgg_keys.json")
CHUNK = os.path.join(HERE, "gbuffer_chunk")
SIZES = ((64, 64), (50, 70))


def reference_lpips_module():
    import torchvision
    tv_vgg16 = torchvision.models.vgg16
    torchvision.models.vgg16 = lambda pretrained=False, **kw: tv_vgg16(weights=None)
    try:
        import requests  # noqa: F401
    except ImportError:
        _ref_stubs.mod("requests")
    import nsr  # noqa: F401  (first: nsr and sgm import each other, and only this order resolves)
    mod = importlib.import_module("sgm.modules.autoencoding.lpips.loss.lpips")
    mod.LPIPS.load_from_pretrained = lambda self, name="vgg_lpips": None
    return mod


def reference_ssim_module():
    """nsr/losses/builder.py.  Its top-level imports reach packages this image lacks beyond _ref_stubs' list
    (torchtyping for annotations, ...); each one reported missing is stubbed and the import retried."""
    class _Subscriptable:
        def __class_getitem__(cls, item):
            return cls
    for _ in range(20):
        try:
            return importlib.import_module("nsr.losses.builder")
        except ModuleNotFoundError as e:
            print("stubbing absent module", e.name)
            _ref_stubs.mod(e.name, TensorType=_Subscriptable)
            for k in [k for k in sys.modules if k.startswith("nsr.losses")]:
                del sys.modules[k]
    raise RuntimeError("nsr.losses.builder does not import")


def chunk_views(h, w):
    from PIL import Image
    a = np.asarray(Image.open(os.path.join(CHUNK, "raw_img.jpg")).convert("RGB"), dtype=np.float32) / 255.0
    S = a.shape[0]
    v = torch.from_numpy(a).reshape(S, -1, S, 3).permute(1, 3, 0, 2)            # [16, 3, S, S]
    return F.interpolate(v[[0, 1, 5]], size=(h, w), mode="area") * 2 - 1


def pairs(h, w, g):
    v = chunk_views(h, w)
    a = v[[0, 0, 1, 2]]
    noisy = (v[0] + 0.05 * 2 * torch.randn(v[0].shape, generator=g)).clamp(-1, 1)   # sigma 0.05 on [0, 1]
    blur = F.avg_pool2d(F.pad(v[1:2], (1, 1, 1, 1), mode="replicate"), 3, 1)[0]
    shift = torch.roll(v[2], shifts=(2, 2), dims=(1, 2))
    b = torch.stack([v[1], noisy, blur, shift])
    return a.contiguous(), b.contiguous()


def main():
    from oracle.lpips_oracle import random_state_dict
    mod = reference_lpips_module()
    model = mod.LPIPS().eval()
    sd_ref = model.state_dict()
    with open(KEYS, "w") as f:
        json.dump({k: list(v.shape) for k, v in sd_ref.items()}, f, indent=1)
    sd = random_state_dict(SEED)
    model.load_state_dict(sd, strict=True)
    builder = reference_ssim_module()
    win = builder.create_window(11, 3)
    captured = []
    avg = mod.spatial_average

    def spatial_average(x, keepdim=True):          # forward adds the later taps into the first one in place: keep copies
        r = avg(x, keepdim)
        captured.append(r.clone())
        return r
    mod.spatial_average = spatial_average
    g = torch.Generator().manual_seed(1)
    out = {"seed": np.int64(SEED)}
    for k in sorted(sd):
        out["sum/" + k] = np.float64(sd[k].double().sum())
        out["first/" + k] = sd[k].reshape(-1)[:4].numpy()
    for h, w in SIZES:
        a, b = pairs(h, w, g)
        captured.clear()
        with torch.no_grad():
            val = model(a, b)
        per = torch.cat([c.reshape(-1, 1) for c in captured], 1)
        s = builder._ssim(((a + 1) / 2).double(), ((b + 1) / 2).double(), win.double(), 11, 3, size_average=False)
        tag = "%dx%d/" % (h, w)
        out.update({tag + "in0": a.numpy(), tag + "in1": b.numpy(), tag + "per_tap": per.numpy(),
                    tag + "value": val.reshape(-1).numpy(), tag + "ssim": s.numpy()})
        print(tag, "lpips", val.reshape(-1).tolist(), "ssim", s.tolist())
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes;", KEYS)


if __name__ == "__main__":
    main()
