"""ctypes binding of libga_b200.so (the C ABI in include/ga_b200.h).

There is NO CPU fallback: if the shared library is missing or does not load,
importing anything that computes raises.  Build it with
`python -m gaussiananything_b200.build` (nvcc, sm_90a).
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# GA_B200_LIB: load a tuning build (gaussiananything_b200/build.py --variant) instead of the product library
LIB_PATH = os.environ.get("GA_B200_LIB") or os.path.join(_HERE, "libga_b200.so")

_lib = None


class GaRasterLayout(C.Structure):
    _fields_ = [(n, C.c_size_t) for n in (
        "total_bytes", "status", "rec", "depth", "rect", "tile_count", "tile_start",
        "keys", "ids", "final_T", "n_contrib", "inst_cnt", "n_list", "tile_flag", "lists")]


class GaGemmEpilogue(C.Structure):
    _fields_ = [("mode", C.c_int), ("bias", C.c_void_p), ("out", C.c_void_p), ("ld_out", C.c_int),
                ("gate", C.c_void_p), ("gate_ld", C.c_int), ("rows_per_batch", C.c_int),
                ("q", C.c_void_p), ("k", C.c_void_p), ("vt", C.c_void_p),
                ("qn_w", C.c_void_p), ("kn_w", C.c_void_p), ("heads", C.c_int), ("first_part", C.c_int),
                ("tok_pitch", C.c_int), ("eps", C.c_float)]


# GaGemmEpilogue.mode: the header's GA_EPI_* (tests/test_abi.py checks them against it)
EPI_BF16, EPI_GELU_BF16, EPI_F32, EPI_RESID_GATE_F32, EPI_HEADS, EPI_GEGLU_BF16 = 0, 1, 2, 3, 4, 5
# ga_linear_grad_validate's op: the header's GA_LINEAR_*
LINEAR_FC1, LINEAR_DGRAD, LINEAR_WGRAD, LINEAR_BGRAD = 0, 1, 2, 3


class GaVaeEncHead(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("ln_w", "ln_b", "fc1_w", "fc1_b", "fc2_w", "fc2_b", "q1_w", "q1_b", "q2_w",
                                          "q2_b")] + [("ln_eps", C.c_float)]


vp, i32, i64, f32, sz = C.c_void_p, C.c_int, C.c_int64, C.c_float, C.c_size_t
_RASTER_IN = [vp, i32, i32, i32, vp, vp, vp, i32, i32, f32]   # gauss13, batch, P, views, viewmats, projmats, bg, H, W, scale

# name: (restype, argtypes) of every function include/ga_b200.h declares, in its order
# (tests/test_abi.py checks this table against the header)
ABI = {
    "ga_raster_layout_ex": (i32, [i32, i32, i32, i32, i32, i64, i32, C.POINTER(GaRasterLayout)]),
    "ga_raster_forward_ex": (i32, _RASTER_IN + [vp, vp, vp, vp, sz, i64, i32, vp, vp, vp]),
    "ga_raster_backward_scratch_bytes": (sz, [i32, i32, i32]),
    "ga_raster_backward_ex": (i32, _RASTER_IN + [vp, vp, vp, vp, sz, i64, i32, vp, sz, vp, vp]),
    "ga_render_post_forward": (i32, [vp, vp, vp, i32, i32, i32, vp, vp, vp, vp, vp, vp]),
    "ga_render_post_backward": (i32, [vp, vp, vp, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp]),
    "ga_raster_set_variant": (i32, [i32, i32]),
    "ga_gemm_bf16_tn": (i32, [vp, i32, vp, i32, i32, i32, i32, C.POINTER(GaGemmEpilogue), i32, vp]),
    "ga_gemm_validate": (i32, [vp, i32, vp, i32, i32, i32, i32, C.POINTER(GaGemmEpilogue), i32]),
    "ga_attention_bf16": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, f32, f32, vp]),
    "ga_attention_causal_bf16": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, f32, f32, vp]),
    "ga_attention_validate": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32]),
    "ga_rmsnorm_modulate": (i32, [vp, vp, vp, vp, i32, i32, vp, i32, i32, f32, vp]),
    "ga_linear_small": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp]),
    "ga_timestep_sinusoid": (i32, [vp, vp, i32, i32, vp]),
    "ga_layernorm_rows": (i32, [vp, vp, vp, vp, i32, i32, f32, vp]),
    "ga_add_tables": (i32, [vp, vp, vp, i32, i32, i32, i32, vp]),
    "ga_embed_fc1": (i32, [vp, i32, vp, i32, vp, vp, vp, i32, i32, vp]),
    "ga_xyz_posenc": (i32, [vp, vp, i32, vp]),
    "ga_final_layer": (i32, [vp, vp, vp, vp, vp, i32, i32, i32, i32, f32, vp]),
    "ga_cfg_combine": (i32, [vp, vp, i64, f32, vp]),
    "ga_axpy": (i32, [vp, vp, f32, i64, vp]),
    "ga_f32_to_bf16": (i32, [vp, vp, i64, vp]),
    "ga_layernorm_modulate": (i32, [vp, vp, vp, vp, vp, i32, i32, vp, i32, i32, f32, vp]),
    "ga_thin_linear": (i32, [vp, vp, vp, i32, vp, vp, vp, i32, i32, i32, f32, vp]),
    "ga_micro_attention_bf16": (i32, [vp, vp, vp, vp, i32, i32, i32, f32, vp]),
    "ga_micro_seq_build": (i32, [vp, i32, vp, vp, i64, i32, i32, vp]),
    "ga_surfel_cascade_pack": (i32, [vp, i32, vp, vp, i32, i32, f32, f32, vp, vp, i64, vp]),
    "ga_silu_to_bf16": (i32, [vp, vp, i64, vp]),
    "ga_dino_frontend_scratch_bytes": (sz, [i32, i32, i32, i32]),
    "ga_dino_frontend": (i32, [vp, i32, i32, i32, i32, i32, vp, i32, vp, sz, vp]),
    "ga_dino_tokens": (i32, [vp, vp, vp, i32, vp, vp, i32, i32, i32, vp]),
    "ga_mesh_work_bytes": (sz, [i64]),
    "ga_mesh_prepare": (i32, [vp, vp, vp, i32, i32, i32, vp, f32, vp, vp]),
    "ga_mesh_touch": (i32, [vp, i32, i32, i32, vp, vp, vp, i32, vp, vp, vp, vp, vp, vp, vp, vp]),
    "ga_mesh_integrate": (i32, [vp, i32, i32, i32, vp, vp, vp, vp, vp, i32, vp, vp]),
    "ga_mesh_cubes_count": (i32, [vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "ga_mesh_cubes_emit": (i32, [vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "ga_mesh_clusters": (i32, [vp, i32, vp, i64, vp, vp, vp, vp, vp, vp, vp]),
    "ga_mesh_filter": (i32, [vp, vp, i32, vp, i32, vp, vp, i32, vp, vp, vp, vp, vp, vp, vp, vp]),
    "ga_conv3x3_out_size": (i32, [i32, i32]),
    "ga_conv3x3_bf16": (i32, [vp, i32, i32, i32, i32, vp, i32, vp, i32, i32, vp, vp, vp, vp]),
    "ga_group_norm_scratch_bytes": (sz, [i32, i32]),
    "ga_group_norm_nhwc": (i32, [vp, vp, vp, i32, i32, i32, f32, i32, vp, i32, vp, sz, vp]),
    "ga_fps": (i32, [vp, i32, i32, i32, vp, vp, vp, vp]),
    "ga_vae_enc_input": (i32, [vp, i32, i32, i32, i32, i32, vp, i32, i32, i32, vp, vp]),
    "ga_heads32_split": (i32, [vp, vp, vp, i32, i32, i32, i32, f32, vp, vp, vp, vp]),
    "ga_vae_enc_head": (i32, [C.POINTER(GaVaeEncHead), vp, vp, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp]),
    "ga_clip_text_embed": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, vp]),
    "ga_clip_text_eot_gather": (i32, [vp, vp, vp, i32, i32, i32, vp]),
    "ga_quick_gelu_bf16": (i32, [vp, i64, vp]),
    "ga_gbuffer_pack": (i32, [vp, vp, vp, vp, vp, i32, i32, i32, vp, i32, vp, vp, vp, vp, vp, vp]),
    "ga_recon_metrics": (i32, [vp, vp, vp, vp, vp, vp, vp, vp, vp, i64, i32, i32, i32, vp, vp, vp]),
    "ga_conv3x3_relu_bf16": (i32, [vp, i32, i32, i32, i32, vp, i32, vp, i32, vp, vp]),
    "ga_lpips_pack": (i32, [vp, vp, i32, i32, i32, i32, vp, vp, vp, vp]),
    "ga_maxpool2x2_bf16": (i32, [vp, i32, i32, i32, i32, vp, vp]),
    "ga_lpips_head": (i32, [vp, i32, i32, i32, i32, vp, vp, vp]),
    "ga_lpips_reduce": (i32, [vp, i32, i32, i32, vp, vp]),
    "ga_ssim_scratch_bytes": (sz, [i32, i32, i32]),
    "ga_ssim": (i32, [vp, vp, i32, i32, i32, vp, vp, sz, vp, vp]),
    "ga_conv3x3_mask_bf16": (i32, [vp, i32, i32, i32, i32, vp, i32, i32, vp, vp, vp]),
    "ga_lpips_tap_backward": (i32, [vp, i32, i32, i32, i32, i32, vp, vp, vp, vp, vp]),
    "ga_lpips_input_backward": (i32, [vp, i32, i32, i32, vp, vp, i32, vp, vp]),
    "ga_fps_ex_workspace_bytes": (sz, [i32, i32, i32]),
    "ga_fps_ex": (i32, [vp, vp, i32, i32, i32, vp, vp, vp, vp, sz, vp]),
    "ga_chunk_surface_points_scratch_bytes": (sz, [i32, i32, i32]),
    "ga_chunk_surface_points": (i32, [vp, vp, vp, i32, i32, i32, vp, i32, i32, f32, vp, vp, vp, sz, vp]),
    "ga_conv4x4_out_size": (i32, [i32, i32]),
    "ga_conv4x4_lrelu_bf16": (i32, [vp, i32, i32, i32, i32, vp, i32, vp, i32, i32, vp, vp]),
    "ga_conv4x4_stats": (i32, [vp, i32, i32, i32, i32, vp, i32, i32, i32, vp, vp, vp]),
    "ga_disc_bn_forward": (i32, [vp, vp, i64, i32, vp, vp, i32, f32, f32, vp, vp, vp, vp, vp, vp]),
    "ga_disc_conv5": (i32, [vp, i32, i32, i32, vp, vp, vp, vp]),
    "ga_disc_conv5_partials": (i32, [i32, i32, i32]),
    "ga_disc_conv5_backward": (i32, [vp, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "ga_disc_dgrad_partials": (i32, [i32, i32, i32, i32]),
    "ga_disc_dgrad": (i32, [vp, i32, i32, i32, i32, vp, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp]),
    "ga_disc_bn_backward": (i32, [vp, vp, i64, i32, vp, vp, vp, vp, i32, i32, vp, vp, vp, vp, vp]),
    "ga_disc_wgrad_workspace_bytes": (sz, [i32, i32, i32, i32, i32]),
    "ga_disc_wgrad": (i32, [vp, vp, i32, i32, i32, i32, i32, i32, i32, vp, sz, vp, vp]),
    "ga_disc_colsum_scratch_bytes": (sz, [i64, i32]),
    "ga_disc_colsum": (i32, [vp, i32, i64, i32, vp, sz, vp, vp]),
    "ga_disc_input_backward": (i32, [vp, i32, i32, i32, vp, vp, vp]),
    "ga_attention_grad_validate": (i32, [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp,
                                         i32]),
    "ga_attention_fwd_lse_bf16": (i32, [vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp, f32, vp]),
    "ga_attention_bwd_bf16": (i32, [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp, f32,
                                    vp]),
    "ga_linear_grad_validate": (i32, [i32, vp, vp, vp, vp, i32, i32, i32, i32, i32, vp, sz]),
    "ga_linear_fc1_gelu_bf16": (i32, [vp, vp, vp, vp, vp, i32, i32, i32, i32, vp]),
    "ga_linear_dgrad_bf16": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, vp]),
    "ga_linear_wgrad_splits": (i32, [i32, i32, i32]),
    "ga_linear_wgrad_workspace_bytes": (sz, [i32, i32, i32]),
    "ga_linear_wgrad_bf16": (i32, [vp, vp, vp, i32, i32, i32, vp, sz, vp]),
    "ga_linear_bias_grad_workspace_bytes": (sz, [i32, i32]),
    "ga_linear_bias_grad_bf16": (i32, [vp, vp, i32, i32, vp, sz, vp]),
    "ga_dit_grad_partials": (i32, [i32, i32]),
    "ga_dit_rmsnorm_bwd_validate": (i32, [vp, vp, vp, vp, i32, vp, vp, vp, vp, vp, i32, i32, i32, i32]),
    "ga_dit_rmsnorm_bwd": (i32, [vp, vp, vp, vp, i32, vp, vp, vp, vp, vp, i32, i32, i32, i32, f32, vp]),
    "ga_dit_gate_bwd_validate": (i32, [vp, vp, vp, i32, vp, vp, i32, i32, i32, i32]),
    "ga_dit_gate_bwd": (i32, [vp, vp, vp, i32, vp, vp, i32, i32, i32, i32, vp]),
    "ga_dit_gate_residual_validate": (i32, [vp, vp, vp, i32, vp, vp, vp, vp, i32, vp, i32, i32, i32]),
    "ga_dit_gate_residual": (i32, [vp, vp, vp, i32, vp, vp, vp, vp, i32, vp, i32, i32, i32, f32, vp]),
    "ga_dit_qk_norm_validate": (i32, [i32, vp, i32, vp, i32, vp, i32, vp, vp, vp, i32, i32, i32]),
    "ga_dit_qk_norm_fwd_bf16": (i32, [vp, i32, vp, i32, vp, vp, i32, i32, i32, f32, vp]),
    "ga_dit_qk_norm_bwd_bf16": (i32, [vp, i32, vp, i32, vp, i32, vp, vp, vp, i32, i32, i32, f32, vp]),
    "ga_dit_grad_reduce_validate": (i32, [vp, vp, i32, i32, i32]),
    "ga_dit_grad_reduce": (i32, [vp, vp, i32, i32, i32, vp]),
    "ga_dit_final_layer_bwd_validate": (i32, [vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32]),
    "ga_dit_final_layer_bwd": (i32, [vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, f32, vp]),
    "ga_dit_embed_fc1_bwd_validate": (i32, [vp, i32, vp, i32, vp, vp, vp, vp, vp, vp, i32, i32]),
    "ga_dit_embed_fc1_bwd": (i32, [vp, i32, vp, i32, vp, vp, vp, vp, vp, vp, i32, i32, vp]),
    "ga_dit_linear_small_bwd_validate": (i32, [vp, i32, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32]),
    "ga_dit_linear_small_bwd": (i32, [vp, i32, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, vp]),
    "ga_dit_layernorm_rows_bwd_validate": (i32, [vp, vp, vp, vp, vp, vp, i32, i32]),
    "ga_dit_layernorm_rows_bwd": (i32, [vp, vp, vp, vp, vp, vp, i32, i32, f32, vp]),
    "ga_profile_enable": (i32, [i32]),
    "ga_profile_read": (i32, [C.POINTER(f32), i32]),
    "ga_b200_version": (C.c_char_p, []),
}


def lib():
    """Returns the loaded library with every function of ABI declared; raises loudly when it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "gaussiananything_b200: %s is missing -- build it with "
            "`python -m gaussiananything_b200.build` (there is no CPU fallback)" % LIB_PATH)
    import torch  # noqa: F401  (loads libcudart / libcuda into the process first)
    L = C.CDLL(LIB_PATH)
    for name, (restype, argtypes) in ABI.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = restype, argtypes
    _lib = L
    return L


def check(rc, what):
    if rc != 0:
        raise RuntimeError("libga_b200: %s failed with code %d" % (what, rc))
