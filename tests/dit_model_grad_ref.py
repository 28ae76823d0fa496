"""fp64 references of the trainable image-to-3D DiT (include/ga_b200.h Part 15, gaussiananything_b200/dit_grad.py
model_forward) for the dit_model_grad tests: torch only, no library import.

model(P, x, t, context, heads, depth, dy) restates oracle/dit_oracle.forward (which tests/test_oracle_dit.py pins to
the reference's own code) under autograd, the blocks by tests/dit_grad_ref.py, in the dtype of the tensors given
(float64 for the references): {y, dx, dctx, dvec, and one entry per parameter name}.  With emulate=True it rounds
where the kernels round: the blocks as tests/dit_grad_ref.py states; the stem's fc1 output e1 = bf16(gelu_tanh(v)),
the fc2 and xyz-projection weights, the positional encoding, and the gradient of fc2's and the projection's output
(the Part 13 GEMMs read bf16(dxres)).  The B-row stem, the LayerNorms, the final layer and all sums stay exact.
"""
import math

import torch
import torch.nn.functional as F

from tests import dit_grad_ref as BR

STEM = ("t_embedder.mlp.0.weight", "t_embedder.mlp.0.bias", "t_embedder.mlp.2.weight", "t_embedder.mlp.2.bias",
        "pooled_vec_embedder.0.weight", "pooled_vec_embedder.0.bias", "pooled_vec_embedder.1.weight",
        "pooled_vec_embedder.1.bias", "adaLN_modulation.1.weight", "adaLN_modulation.1.bias",
        "x_embedder.fc1.weight", "x_embedder.fc1.bias", "x_embedder.fc2.weight", "x_embedder.fc2.bias")
PE = ("xyz_pos_embed.xyz_projection.weight", "xyz_pos_embed.xyz_projection.bias")
HEAD = ("final_layer.scale_shift_table", "final_layer.linear.weight", "final_layer.linear.bias")


def param_names(sd, depth):
    names = STEM + (PE if PE[0] in sd else ()) + HEAD
    return names + tuple("blocks.%d.%s" % (l, k) for l in range(depth) for k in BR.PARAMS)


def timestep_embedding(t, dim=256):
    half = dim // 2
    freqs = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float64, device=t.device) / half)
    args = t[:, None].double() * freqs[None]
    return torch.cat([torch.cos(args), torch.sin(args)], -1).to(t.dtype if t.is_floating_point() else torch.float64)


def xyz_posenc(xyz):
    out = [xyz]
    for k in range(10):
        out += [torch.sin(xyz * 2.0 ** k), torch.cos(xyz * 2.0 ** k)]
    return torch.cat(out, -1)


def stem(P, x, t, vec, xyz, rounding=False):
    """(xres [B, N, D], t0 [B, 6 D], temb [B, D])"""
    rf, rg = (BR._rf, BR._RoundGrad.apply) if rounding else ((lambda u: u),) * 2
    sinus = timestep_embedding(t.reshape(-1).expand(x.shape[0]) if t.numel() == 1 else t.reshape(-1)).to(x.dtype)
    a1 = F.linear(sinus, P["t_embedder.mlp.0.weight"], P["t_embedder.mlp.0.bias"])
    temb = F.linear(F.silu(a1), P["t_embedder.mlp.2.weight"], P["t_embedder.mlp.2.bias"])
    vln = F.layer_norm(vec, vec.shape[-1:], P["pooled_vec_embedder.0.weight"], P["pooled_vec_embedder.0.bias"], 1e-5)
    temb = temb + F.linear(vln, P["pooled_vec_embedder.1.weight"], P["pooled_vec_embedder.1.bias"])
    t0 = F.linear(F.silu(temb), P["adaLN_modulation.1.weight"], P["adaLN_modulation.1.bias"])
    use_pe = PE[0] in P
    xin = torch.cat([xyz, x], -1) if (xyz is not None and not use_pe) else x
    e1 = rf(F.gelu(F.linear(xin, P["x_embedder.fc1.weight"], P["x_embedder.fc1.bias"]), approximate="tanh"))
    xres = rg(F.linear(e1, rf(P["x_embedder.fc2.weight"]), P["x_embedder.fc2.bias"]))
    if use_pe:
        pe = rf(xyz_posenc(xyz)).detach()
        xres = xres + rg(F.linear(pe, rf(P[PE[0]]), P[PE[1]]))
    return xres, t0, temb


def head(P, h, temb):
    shift, scale = (P["final_layer.scale_shift_table"][None] + temb[:, None]).chunk(2, dim=1)
    y = F.layer_norm(h, h.shape[-1:], None, None, 1e-6) * (1 + scale) + shift
    return F.linear(y, P["final_layer.linear.weight"], P["final_layer.linear.bias"])


def forward(P, x, t, context, heads, depth, rounding=False):
    xyz = context.get("fps-xyz")
    h, t0, temb = stem(P, x, t, context["img_vector"], xyz, rounding)
    for l in range(depth):
        pre = "blocks.%d." % l
        h = BR._block_emu({k: P[pre + k] for k in BR.PARAMS}, h, t0, context["img_crossattn"], heads,
                          rounding=rounding)
    return head(P, h, temb)


def model(sd, x, t, context, heads, depth, dy, emulate=False):
    """{name: fp64 tensor}: y and the gradients of x, img_crossattn (dctx), img_vector (dvec) and every parameter,
    on the device the tensors are on."""
    leaves = {k: sd[k].detach().double().clone().requires_grad_(True) for k in param_names(sd, depth)}
    xs = [v.detach().double().clone().requires_grad_(True) for v in (x, context["img_crossattn"],
                                                                       context["img_vector"])]
    ctx = {"img_crossattn": xs[1], "img_vector": xs[2]}
    if "fps-xyz" in context:
        ctx["fps-xyz"] = context["fps-xyz"].detach().double()
    with torch.enable_grad():
        y = forward(leaves, xs[0], t.detach().double(), ctx, heads, depth, rounding=emulate)
        y.backward(dy.double())
    out = dict(y=y.detach(), dx=xs[0].grad, dctx=xs[1].grad, dvec=xs[2].grad)
    out.update({k: v.grad for k, v in leaves.items()})
    return out


rel_l2 = BR.rel_l2
