"""Mirror of /root/reference/nsr/gs_surfel.py `GaussianRenderer2DGS` (lines 21-202).

Same constructor, attributes and `render(...)` signature / return dict, but the
B x V Python loop (reference lines 65-176: >= 6 launches + one device-to-host
read per view) is a single batched launch set of the CUDA kernels; the
per-view post-processing (reference lines 121-163) is applied to the whole
[B,V,...] batch at once.
"""
import torch

from . import raster as _raster


class GaussianRenderer2DGS:
    def __init__(self, output_size, out_chans, rendering_kwargs, **kwargs):
        if not torch.cuda.is_available():
            raise RuntimeError("GaussianRenderer2DGS needs a CUDA device (reference hard-codes device='cuda', "
                               "nsr/gs_surfel.py:25); there is no CPU fallback")
        self.bg_color = torch.tensor([1, 1, 1], dtype=torch.float32, device="cuda")
        self.output_size = output_size
        self.out_chans = out_chans
        self.rendering_kwargs = rendering_kwargs

    def render(self, gaussians, cam_view, cam_view_proj, cam_pos, tanfov, bg_color=None,
               scale_modifier=1, output_size=None):
        # gaussians: [B, N, 13]; cam_view, cam_view_proj: [B, V, 4, 4]; cam_pos: [B, V, 3]
        if output_size is None:
            output_size = self.output_size
        B, V = cam_view.shape[:2]
        assert gaussians.shape[2] == 13  # scale with 2dof
        gaussians = gaussians.contiguous().float()  # gs rendering in fp32
        if bg_color is None:
            bg_color = self.bg_color
        cam_view = cam_view.float()
        color, allmap, _radii = _raster.rasterize_surfels_batched(
            gaussians, cam_view, cam_view_proj.float(), bg_color, int(output_size), int(output_size),
            float(scale_modifier))
        # alpha / camera->world normals / nan-safe median depth / distortion / clamped image (reference :121-163),
        # one fused kernel for all views instead of ~10 torch kernels per view
        images, alphas, depths, normals, dists = _raster.render_postprocess(color, allmap, cam_view)
        return {
            "image": images,            # [B, V, 3, H, W]
            "alpha": alphas,            # [B, V, 1, H, W]
            "depth": depths,
            "rend_normal": normals,
            "dist": dists,
        }
