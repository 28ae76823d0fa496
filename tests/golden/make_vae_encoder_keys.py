"""Writes tests/golden/vae_encoder_keys.json: {key: shape} of the reference AE checkpoint entries the 3D VAE encoder
reads -- the state_dict of the reference's own HybridEncoderPCDStructuredLatentSNoPCD at the deployed configuration
(shell_scripts/release/inference/vae-3d.sh, nsr/script_util.py:1335-1444) under "encoder.", plus the decoder's
quant_conv (vit/vit_triplane.py:1319-1322) under "decoder.superresolution.".  Run on the build container, where the
reference tree and tests/golden/_ref_stubs.py are available:

    python tests/golden/make_vae_encoder_keys.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _ref_stubs  # noqa: E402,F401  (reference on sys.path, absent third-party packages stubbed)

import torch.nn as nn  # noqa: E402


def reference_keys():
    from nsr.srt.encoder import HybridEncoderPCDStructuredLatentSNoPCD
    from vit.vit_triplane import approx_gelu
    from timm.models.vision_transformer import Mlp
    enc = HybridEncoderPCDStructuredLatentSNoPCD(
        num_frames=8, latent_num=768, double_z=True, resolution=256, in_channels=15, ch=64, ch_mult=[1, 2, 4, 4],
        num_res_blocks=1, dropout=0.0, attn_resolutions=[], out_ch=3, z_channels=10,
        attn_kwargs={"n_heads": 8, "d_head": 64}, attn_type="mv-vanilla")
    keys = {"encoder." + k: list(v.shape) for k, v in enc.state_dict().items()}
    qc = Mlp(in_features=20, out_features=20, act_layer=approx_gelu, drop=0)
    keys.update({"decoder.superresolution.quant_conv." + k: list(v.shape) for k, v in qc.state_dict().items()})
    return enc, keys


if __name__ == "__main__":
    _, keys = reference_keys()
    with open(os.path.join(HERE, "vae_encoder_keys.json"), "w") as f:
        json.dump(keys, f, indent=0, sort_keys=True)
    print(len(keys), "keys")
