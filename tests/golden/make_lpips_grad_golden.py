"""Writes tests/golden/lpips_grad_small.npz (+ .part2.npz) from the reference's own LPIPS module, with autograd.

The module is the reference's sgm/modules/autoencoding/lpips/loss/lpips.py, built as make_lpips_golden.py builds it
(nothing fetched; the seeded random weights oracle.lpips_oracle.random_state_dict(SEED) loaded strictly), then run in
fp64 on the CPU.  Its VGG uses in-place ReLUs, and its normalize_tensor divides by the norm plus 1e-10, so the stored
gradients are what torch autograd gives for the reference's own graph.

Inputs: the in0 / in1 pairs of lpips_small.npz (read from it, not stored again), 64 x 64 and 50 x 70 (the pools drop
rows and columns there).  Per-pair upstream weights G (one of them 0).  Stored per size: g [N] and grad0, grad1
[N, 3, H, W] fp64, d(sum_i g_i LPIPS_i) / d in0 and / d in1.  The 50 x 70 arrays go to the .part2 file (each part
stays under 1 MB).

    python tests/golden/make_lpips_grad_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import make_lpips_golden as base  # noqa: E402
from oracle.golden_io import save_parts  # noqa: E402
from oracle.lpips_oracle import random_state_dict  # noqa: E402

OUT = os.path.join(HERE, "lpips_grad_small.npz")
INPUTS = os.path.join(HERE, "lpips_small.npz")
G = (0.75, -1.25, 0.0, 2.0)


def main():
    mod = base.reference_lpips_module()
    model = mod.LPIPS().eval()
    model.load_state_dict(random_state_dict(base.SEED), strict=True)
    model = model.double()
    g = torch.tensor(G, dtype=torch.float64)
    out, part2 = {"seed": np.int64(base.SEED)}, []
    with np.load(INPUTS) as z:
        for h, w in base.SIZES:
            tag = "%dx%d/" % (h, w)
            a = torch.from_numpy(z[tag + "in0"]).double().requires_grad_(True)
            b = torch.from_numpy(z[tag + "in1"]).double().requires_grad_(True)
            val = model(a, b).reshape(-1)
            ga, gb = torch.autograd.grad((val * g).sum(), [a, b])
            out.update({tag + "g": g.numpy(), tag + "value": val.detach().numpy(), tag + "grad0": ga.numpy(),
                        tag + "grad1": gb.numpy()})
            if (h, w) != base.SIZES[0]:
                part2 += [tag + k for k in ("g", "value", "grad0", "grad1")]
            print(tag, "lpips", val.tolist(), "|grad0|", float(ga.norm()), "|grad1|", float(gb.norm()))
    save_parts(OUT, out, part2)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
