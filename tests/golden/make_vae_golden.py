"""Generates tests/golden/vae_decoder_small.npz by running the REFERENCE's own VAE decode path
(/root/reference/vit/vit_triplane.py `pcd_structured_latent_space_vae_decoder_cascaded`: post_quant_conv ->
dit/dit_decoder.py DiT2 -> conv_sr -> three cascaded up-samplers (nsr/srt/layers.py Transformer) -> activations) on CPU in
fp32, at a small width (the class ties token count to width: N = D = 64 tokens; DiT2 depth 2, 1 head of 64;
cascade factors 8 * 4 * 3 as deployed).  Third-party stubs: _ref_stubs.py.  Zero / constant-initialised parameters
(adaLN, the 13-channel heads) are re-randomised so that every stage contributes; weights are rounded to bf16 and
stored as bf16 bit patterns (uint16).  Build container only.
    python tests/golden/make_vae_golden.py
"""
import contextlib
import io
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from _ref_stubs import *  # noqa: F401,F403  (installs the stubs, puts /root/reference on sys.path)
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from oracle.golden_io import save_parts  # noqa: E402
import torch

from guided_diffusion import dist_util
dist_util.dev = lambda: torch.device("cpu")
from dit import dit_decoder
from dit.dit_models_xformers import DiTBlock
from vit import vit_triplane as vt

OUT = os.path.dirname(os.path.abspath(__file__))
D, DEPTH, HEADS, TOK, ZC = 64, 2, 1, 4, 10
RK = dict(sampler_bbox_min=-0.45, sampler_bbox_max=0.45, z_near=0.01, z_far=100)


def build(seed=0):
    torch.manual_seed(seed)
    with contextlib.redirect_stdout(io.StringIO()):
        dec = dit_decoder.DiT2(input_size=TOK, patch_size=1, in_channels=D, hidden_size=D, depth=DEPTH, num_heads=HEADS,
                               num_classes=0, learn_sigma=False, mixed_prediction=False, context_dim=None, roll_out=True,
                               plane_n=1, return_all_layers=False, in_plane_attention=False, vit_blk=DiTBlock)
        gs = type("G", (), {"rendering_kwargs": RK})()           # the renderer object is only asked for its kwargs
        m = vt.pcd_structured_latent_space_vae_decoder_cascaded(dec, gs, cls_token=False, ldm_z_channels=ZC,
                                                                ldm_embed_dim=ZC, plane_n=1, vae_dit_token_size=TOK,
                                                                sr_ratio=2, vae_p=1)
    g = torch.Generator().manual_seed(seed + 1)
    for n, p in m.named_parameters():
        if float(p.detach().abs().sum()) == 0 or "gaussian_pred" in n or "gaussian_residual_pred" in n or "adaLN" in n:
            p.data.copy_(torch.randn(p.shape, generator=g) * 0.05)
        if "norm" in n and n.endswith(".weight"):
            p.data.copy_(1.0 + 0.1 * torch.randn(p.shape, generator=g))
        p.data.copy_(p.data.to(torch.bfloat16).to(torch.float32))      # exactly bf16-representable
    return m.eval(), g


def main():
    m, g = build()
    B, N = 2, D
    lat = torch.randn(B, N, ZC, generator=g)
    xyz = (torch.rand(B, N, 3, generator=g) - 0.5) * 0.8
    ret = {"latent_normalized": lat, "query_pcd_xyz": xyz}
    with torch.no_grad():
        latent = m.vit_decode_backbone(ret, 64)
        base_pre = m.superresolution["conv_sr"](latent["latent_from_vit"])
        out = m.vit_decode_postprocess(latent, dict(ret))
        fin = m.forward_gaussians(dict(out))
    save = {"meta": np.array([D, DEPTH, HEADS, ZC, B, N], np.int64),
            "scene_range_max": np.float32(RK["sampler_bbox_max"]), "skip_weight": np.float32(float(m.skip_weight)),
            "in_latent": lat.numpy(), "in_xyz": xyz.numpy(),
            "out_post_quant": latent["latent"].numpy(), "out_latent_from_vit": latent["latent_from_vit"].numpy(),
            "out_base_pre_activate": base_pre.numpy(), "out_gaussians_base": out["gaussians_base"].numpy(),
            "out_gaussians_upsampled": out["gaussians_upsampled"].numpy(),
            "out_gaussians_upsampled_2": out["gaussians_upsampled_2"].numpy(),
            "out_gaussians_upsampled_3": out["gaussians_upsampled_3"].numpy(),
            "out_gaussians": fin["gaussians"].numpy()}
    for k, v in m.state_dict().items():
        if v.dtype == torch.float32 and v.numel() > 1:
            save["w:" + k] = v.to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)    # bf16 bit pattern
        else:
            save["f:" + k] = v.float().numpy()
    path = os.path.join(OUT, "vae_decoder_small.npz")
    save_parts(path, save, {"out_gaussians_upsampled_2", "out_gaussians_upsampled_3"})     # every file under 1 MB
    print(path, "params", sum(p.numel() for p in m.parameters()), "kB", os.path.getsize(path) // 1024,
          {k: save[k].shape for k in save if k.startswith("out_")})


if __name__ == "__main__":
    main()
