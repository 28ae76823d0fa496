"""Generates tests/golden/dit_*.npz by running the REFERENCE's own DiT and
transport code (/root/reference/dit/dit_i23d.py, dit/dit_models_xformers.py,
vit/vision_transformer.py, ldm/modules/attention.py, dit/norm.py, transport/*)
on CPU in fp32.  Third-party packages that are absent from this image are
replaced by stubs that restate their published semantics:
  * xformers.ops.memory_efficient_attention == softmax(q k^T / sqrt(d)) v  (-> torch SDPA)
  * xformers FusedMLP == Linear(no bias) -> +bias -> exact GELU -> Linear(no bias) -> +bias,
    state-dict keys mlp.mlp.{0.weight,1.bias,2.weight,3.bias}
  * timm Mlp / PatchEmbed; torchdiffeq.odeint fixed-grid euler/midpoint/heun/rk4
  * everything else missing (kiui, pytorch3d, ...) is a dummy: never on this path.
Only runs inside the build container (needs /root/reference); the .npz files it
writes are committed and are what tests/ read.  Weights are stored as bf16 bit
patterns (every value is exactly bf16-representable).
    python tests/golden/make_dit_golden.py
"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from _ref_stubs import *  # noqa: F401,F403  (installs the stubs, exposes torch / nn / F / mod)
import torch, torch.nn as nn, torch.nn.functional as F
import io, contextlib, os
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from oracle.golden_io import save_parts  # noqa: E402
from dit import dit_i23d, dit_models_xformers as dmx
import transport as ref_transport

OUT = os.path.dirname(os.path.abspath(__file__))
UNUSED = ("clip_spatial_proj.", "cap_embedder.", "attention_y_norm.")


def bf16_round_(t):
    t.data.copy_(t.data.to(torch.bfloat16).to(torch.float32))


def build(cls, seed, **kw):
    torch.manual_seed(seed)
    with contextlib.redirect_stdout(io.StringIO()):
        m = cls(patch_size=1, vit_blk=dmx.ImageCondDiTBlockPixelArtRMSNormClayLRM, use_clay_ca=True,
                input_size=32, num_classes=0, learn_sigma=False, roll_out=True, pooling_ctx_dim=768, **kw)
    g = torch.Generator().manual_seed(seed + 1)
    for n, p in m.named_parameters():
        # the reference zero-initialises these (dit_i23d.py:213-214,508-509; dit_models_xformers.py:1158-1159):
        # re-randomise so the output is not identically zero (SURVEY.md 8d); also make norm gains non-trivial
        if n.startswith(("final_layer.linear", "adaLN_modulation", "pooled_vec_embedder.1")) or n.endswith(".bias"):
            p.data.copy_(torch.randn(p.shape, generator=g) * 0.02)
        if "norm" in n and n.endswith(".weight"):
            p.data.copy_(1.0 + 0.1 * torch.randn(p.shape, generator=g))
        bf16_round_(p)
    return m.eval()


def run(name, cls, seed, B, N, M, Cin, ctx_dim, stage2, **kw):
    m = build(cls, seed, in_channels=Cin, context_dim=ctx_dim, **kw)
    g = torch.Generator().manual_seed(100 + seed)
    x = torch.randn(2 * B, N, Cin, generator=g)
    t = torch.rand(2 * B, generator=g)
    ctx = {"img_crossattn": torch.randn(2 * B, M, ctx_dim, generator=g),
           "img_vector": torch.randn(2 * B, ctx_dim, generator=g)}
    if stage2:
        ctx["fps-xyz"] = torch.rand(2 * B, N, 3, generator=g) * 2 - 1
    acts = {}
    hooks = [blk.register_forward_hook(lambda mod, a, out, i=i: acts.__setitem__("block%d" % i, out.detach().clone()))
             for i, blk in enumerate(m.blocks)]
    with torch.no_grad():
        y = m(x, t, ctx)
        y_cfg = m.forward_with_cfg(x, t, ctx, 4.0)
        for h in hooks:
            h.remove()
        tr = ref_transport.create_transport("GVP", "velocity", None, None, None, "lognorm")
        sampler = ref_transport.Sampler(tr)
        traj_euler = sampler.sample_ode(sampling_method="euler", num_steps=5)(x, m.forward_with_cfg, context=ctx, cfg_scale=4.0)
        traj_heun = sampler.sample_ode(sampling_method="heun2", num_steps=4)(x, m.forward_with_cfg, context=ctx, cfg_scale=4.0)
    sd = {k: v for k, v in m.state_dict().items() if not any(u in k for u in UNUSED)}
    save = {"sd__" + k: v.to(torch.bfloat16).view(torch.int16).numpy() for k, v in sd.items()}
    for k, v in sd.items():
        assert torch.equal(v.to(torch.bfloat16).to(torch.float32), v), k
    save.update(x=x.numpy(), t=t.numpy(), y=y.numpy(), y_cfg=y_cfg.numpy(),
                traj_euler=traj_euler.numpy(), traj_heun=traj_heun.numpy(),
                **{"ctx__" + k: v.numpy() for k, v in ctx.items()},
                **{"act__" + k: v.numpy() for k, v in acts.items()})
    save["meta"] = np.array([kw["depth"], kw["hidden_size"], kw["num_heads"], Cin, ctx_dim, int(stage2),
                             int(kw.get("use_pe_cond", False))])
    # the second block's weights go to <name>.part2.npz: every committed file stays under 1 MB
    save_parts(os.path.join(OUT, name + ".npz"), save, {k for k in save if k.startswith("sd__blocks.1.")})
    print(name, "params", sum(v.numel() for v in sd.values()), "|y|", float(y.abs().mean()))


run("dit_stage1_small", dit_i23d.DiT_I23D_PCD_PixelArt_noclip, 1, B=1, N=24, M=10, Cin=3, ctx_dim=64, stage2=False,
    depth=2, hidden_size=128, num_heads=2)
run("dit_stage2_small", dit_i23d.DiT_I23D_PCD_PixelArt_noclip_clay_stage2, 2, B=1, N=16, M=7, Cin=10, ctx_dim=32,
    stage2=True, depth=1, hidden_size=64, num_heads=1, use_pe_cond=True)
# stage 2 in concatenation mode (x_embedder sees cat([fps_xyz, x]); the stage2-B registry entry uses it)
run("dit_stage2_concat_small", dit_i23d.DiT_I23D_PCD_PixelArt_noclip_clay_stage2, 3, B=2, N=20, M=9, Cin=10, ctx_dim=32,
    stage2=True, depth=1, hidden_size=64, num_heads=1, use_pe_cond=False)
