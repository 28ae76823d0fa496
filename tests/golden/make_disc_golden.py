"""Writes tests/golden/disc_small.npz (+ .part2.npz) and tests/golden/disc_keys.json from the reference's own
nsr/losses/disc.py NLayerDiscriminator(input_nc=3, ndf=64, n_layers=3, use_actnorm=False), run in fp64 on the CPU
with gaussiananything_b200.disc.random_state_dict(SEED) loaded strictly.  Its `.util` import (ActNorm, unused at
use_actnorm=False) is stubbed.  Build container only: it reads the reference tree.

Inputs: the first four views of the committed G-buffer chunk (tests/golden/gbuffer_chunk/raw_img.jpg) in [-1, 1],
area-resized to 64 x 64 and to 50 x 70 (the real batch), and the real batch plus 0.1 N(0, 1) noise (the fake batch).
Protocol per size, in training mode: logits of the real call, then of the fake call (two BatchNorm batches);
hinge_d_loss (nsr/losses/vqperceptual.py) of the two; the running statistics after both calls; the parameter
gradients of the d-loss; the g-loss -mean(fake logits) and its gradient to the fake images; then eval-mode logits of
the real batch.  Parameter gradients are stored at every STRIDE-th element (flattened) plus each tensor's sum and L2
norm.  The 50 x 70 arrays go to the .part2 file (each part stays under 1 MB).

    python tests/golden/make_disc_golden.py
"""
import importlib.util
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from gaussiananything_b200 import disc  # noqa: E402
from gaussiananything_b200.gbuffer import read_chunk  # noqa: E402
from oracle.golden_io import save_parts  # noqa: E402

REF = "/root/reference/nsr/losses/disc.py"
OUT = os.path.join(HERE, "disc_small.npz")
KEYS = os.path.join(HERE, "disc_keys.json")
SEED = 20261017
SIZES = ((64, 64), (50, 70))
VIEWS = 4
STRIDE = 997


def reference_module():
    pkg = types.ModuleType("nsr_losses_stub")
    pkg.__path__ = []
    util = types.ModuleType("nsr_losses_stub.util")
    util.ActNorm = None
    sys.modules["nsr_losses_stub"] = pkg
    sys.modules["nsr_losses_stub.util"] = util
    spec = importlib.util.spec_from_file_location("nsr_losses_stub.disc", REF)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def inputs(h, w):
    ch = read_chunk(os.path.join(HERE, "gbuffer_chunk"))
    img = ch["raw_img"]
    n = ch["depth"].shape[0]
    vw = img.shape[1] // n
    views = np.stack([img[:, i * vw:(i + 1) * vw] for i in range(VIEWS)]).astype(np.float64) / 127.5 - 1.0
    t = torch.from_numpy(views).permute(0, 3, 1, 2)
    real = F.interpolate(t, size=(h, w), mode="area")
    g = torch.Generator().manual_seed(SEED + h * 1000 + w)
    fake = real + 0.1 * torch.randn(real.shape, generator=g, dtype=torch.float64)
    return real.float().double(), fake.float().double()


def hinge_d_loss(logits_real, logits_fake):          # nsr/losses/vqperceptual.py
    return 0.5 * (torch.mean(F.relu(1.0 - logits_real)) + torch.mean(F.relu(1.0 + logits_fake)))


def main():
    mod = reference_module()
    out, part2 = {"seed": np.int64(SEED), "stride": np.int64(STRIDE)}, []
    m = mod.NLayerDiscriminator(input_nc=3, ndf=64, n_layers=3, use_actnorm=False)
    with open(KEYS, "w") as f:
        json.dump({k: list(v.shape) for k, v in m.state_dict().items()}, f, indent=1)
    for h, w in SIZES:
        tag = "%dx%d/" % (h, w)
        m = mod.NLayerDiscriminator(input_nc=3, ndf=64, n_layers=3, use_actnorm=False)
        m.load_state_dict(disc.random_state_dict(SEED), strict=True)
        m = m.double().train()
        real, fake = inputs(h, w)
        fake = fake.requires_grad_(True)
        lr = m(real)
        lf = m(fake)
        d_loss = hinge_d_loss(lr, lf)
        params = [p for _, p in m.named_parameters()]
        names = [k for k, _ in m.named_parameters()]
        gp = torch.autograd.grad(d_loss, params, retain_graph=True)
        g_loss = -torch.mean(lf)
        gx, = torch.autograd.grad(g_loss, [fake])
        rec = {"real": real.float().numpy(), "fake": fake.detach().float().numpy(), "logits_real": lr.detach().numpy(),
               "logits_fake": lf.detach().numpy(), "d_loss": d_loss.detach().numpy(), "g_loss": g_loss.detach().numpy(),
               "grad_fake": gx.numpy()}
        for k, v in m.state_dict().items():
            if "running" in k or "num_batches" in k:
                rec["state/" + k] = v.numpy()
        for k, g in zip(names, gp):
            flat = g.reshape(-1)
            rec["grad/%s/strided" % k] = flat[::STRIDE].numpy()
            rec["grad/%s/sum" % k] = flat.sum().numpy()
            rec["grad/%s/norm" % k] = flat.norm().numpy()
        m.eval()
        with torch.no_grad():
            rec["logits_eval"] = m(real).numpy()
        for k, v in rec.items():
            out[tag + k] = v
            if (h, w) != SIZES[0]:
                part2.append(tag + k)
        print(tag, "d_loss", float(d_loss), "g_loss", float(g_loss), "|grad_fake|", float(gx.norm()))
    save_parts(OUT, out, part2)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
