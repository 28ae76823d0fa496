"""Writes tests/golden/vae_encoder_small{,.part2}.npz from the reference's own HybridEncoderPCDStructuredLatentSNoPCD and the
posterior of vit/vit_triplane.py:1347-1385, on CPU in fp32, at the deployed widths (ch 64, so GroupNorm(32), the
8 x 64 and 8 x 32 heads are real) on a small shape: B = 1, V = 2 views of 64^2 (2 x 64 tokens), 512 points, K = 64.

The weights are not stored: they are gaussiananything_b200.vae_encoder.random_state_dict(seed=SEED), re-created by
the test.  pytorch3d's sample_farthest_points / masked_gather are restated here with the start index pinned and the
distance rounding and tie rule the library states (fp32 (dx*dx + dy*dy) + dz*dz, ties to the lowest index); kornia's
BlurPool2D is constructed but unused in forward (the generic stub stands in).

    python tests/golden/make_vae_encoder_golden.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import _ref_stubs  # noqa: E402

SEED, B, V, H, NP, K = 7, 1, 2, 64, 512, 64
START = [123]


def sample_farthest_points(points, lengths=None, K=50, random_start_point=False):
    B_, N, _ = points.shape
    idx = torch.zeros(B_, K, dtype=torch.int64)
    for b in range(B_):
        P = points[b].float()
        md = torch.full((N,), float("inf"))
        cur = START[b] if random_start_point else 0
        for k in range(K):
            idx[b, k] = cur
            if k + 1 == K:
                break
            d = P - P[cur]
            dist = d[:, 0] * d[:, 0]
            dist = dist + d[:, 1] * d[:, 1]
            dist = dist + d[:, 2] * d[:, 2]
            md = torch.minimum(md, dist)
            cur = int(torch.argmax(md))
    return masked_gather(points, idx), idx


def masked_gather(points, idx):
    return torch.gather(points, 1, idx[..., None].expand(*idx.shape, points.shape[-1]))


_ref_stubs.mod("pytorch3d")
_ref_stubs.mod("pytorch3d.ops", sample_farthest_points=sample_farthest_points)
_ref_stubs.mod("pytorch3d.ops.utils", masked_gather=masked_gather)


def main():
    from make_vae_encoder_keys import reference_keys
    from gaussiananything_b200.vae_encoder import random_state_dict
    from torch_utils.distributions.distributions import DiagonalGaussianDistribution
    from einops import rearrange
    enc, _ = reference_keys()
    enc.num_frames, enc.latent_num = V, K
    sd = random_state_dict(seed=SEED)
    enc.load_state_dict({k[len("encoder."):]: v for k, v in sd.items() if k.startswith("encoder.")}, strict=True)
    enc.eval()
    q = "decoder.superresolution.quant_conv."
    from timm.models.vision_transformer import Mlp
    from vit.vit_triplane import approx_gelu
    qc = Mlp(in_features=20, out_features=20, act_layer=approx_gelu, drop=0)
    qc.load_state_dict({k[len(q):]: v for k, v in sd.items() if k.startswith(q)}, strict=True)
    g = torch.Generator().manual_seed(SEED)
    img = torch.randn(B * V, 15, H, H, generator=g)
    pcd = torch.rand(B, NP, 3, generator=g) - 0.5
    eps = torch.randn(B, 10, K, generator=g)
    acts = {}
    hook = lambda name: (lambda m, i, o: acts.__setitem__(name, o.detach().clone()))
    for i in range(4):
        enc.down[i].block[0].register_forward_hook(hook("level%d" % i))
    enc.mid.attn_1.register_forward_hook(hook("attn_1"))
    enc.agg_ca.register_forward_hook(hook("agg_ca"))
    enc.srt.transformer.register_forward_hook(hook("srt"))
    with torch.no_grad():
        out = enc(img, pcd)
        moments = rearrange(qc(out["h"]), "B L C -> B C L")
        post = DiagonalGaussianDistribution(moments, soft_clamp=True)
        latent = rearrange(post.mean + post.std * eps, "B C L -> B L C")
    res = {"img": img, "pcd": pcd, "start": torch.tensor(START), "eps": eps.transpose(1, 2), "h": out["h"],
           "query_pcd_xyz": out["query_pcd_xyz"], "mean": post.mean.transpose(1, 2), "logvar": post.logvar.transpose(1, 2),
           "latent_normalized": latent}
    res.update({"act_" + k: v for k, v in acts.items()})
    arr = {k: v.numpy().astype(np.float32) if v.is_floating_point() else v.numpy() for k, v in res.items()}
    arr["cfg"] = np.array([SEED, B, V, H, NP, K])
    # each file stays below 1 MB: the three largest level outputs are kept at every other row and column
    big = {k: arr.pop(k)[:, :, ::2, ::2] for k in ("act_level0", "act_level1", "act_level2")}
    np.savez_compressed(os.path.join(HERE, "vae_encoder_small.npz"), **arr)
    np.savez_compressed(os.path.join(HERE, "vae_encoder_small.part2.npz"), **big)
    print({k: v.shape for k, v in {**arr, **big}.items()})


if __name__ == "__main__":
    main()
