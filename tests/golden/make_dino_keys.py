"""Writes dinov2_vitl14_reg4_keys.json: the key -> shape table of the torch.hub `dinov2_vitl14_reg` checkpoint
(dinov2_vitl14_reg4_pretrain.pth), the table a real checkpoint must match to load into gaussiananything_b200.dino.

[UPSTREAM-MEMORY] written from the published architecture of DINOv2 ViT-L/14 with registers (facebookresearch/dinov2,
dinov2/models/vision_transformer.py and layers/*, hub entry built with block_chunks=0): embed_dim 1024, depth 24,
16 heads, mlp_ratio 4, 4 register tokens, patch 14, img_size 518 (37 x 37 patches + cls in pos_embed), qkv and
proj with bias, LayerScale on both residual branches, a final LayerNorm; mask_token [1, D].  Not produced by the
reference's code (the hub model is not installed here).  Used by tests/test_dino_cpu.py: the random weights and
the strict loader of gaussiananything_b200.dino are checked against it.

    python tests/golden/make_dino_keys.py
"""
import json
import os

D, DEPTH, MLP, REG, PATCH, GRID = 1024, 24, 4096, 4, 14, 37


def table():
    t = {"cls_token": [1, 1, D], "pos_embed": [1, 1 + GRID * GRID, D], "register_tokens": [1, REG, D],
         "mask_token": [1, D], "patch_embed.proj.weight": [D, 3, PATCH, PATCH], "patch_embed.proj.bias": [D],
         "norm.weight": [D], "norm.bias": [D]}
    for i in range(DEPTH):
        b = "blocks.%d." % i
        for n in ("norm1", "norm2"):
            t[b + n + ".weight"], t[b + n + ".bias"] = [D], [D]
        t[b + "attn.qkv.weight"], t[b + "attn.qkv.bias"] = [3 * D, D], [3 * D]
        t[b + "attn.proj.weight"], t[b + "attn.proj.bias"] = [D, D], [D]
        t[b + "ls1.gamma"], t[b + "ls2.gamma"] = [D], [D]
        t[b + "mlp.fc1.weight"], t[b + "mlp.fc1.bias"] = [MLP, D], [MLP]
        t[b + "mlp.fc2.weight"], t[b + "mlp.fc2.bias"] = [D, MLP], [D]
    return dict(sorted(t.items()))


if __name__ == "__main__":
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "dinov2_vitl14_reg4_keys.json")
    with open(out, "w") as f:
        json.dump(table(), f, indent=0)
        f.write("\n")
    print(out)
