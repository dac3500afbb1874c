"""Autograd boundary of the surfel (2D Gaussian) rasterizer: the interface of `diff_surfel_rasterization`, the package
gaustudio's `surfel_renderer` (configs/2dgs.yaml) imports, on top of the CUDA kernels of csrc/gsr_surfel.cu.

Same public names as the 3DGS module (`GaussianRasterizationSettings`, `GaussianRasterizer`, `rasterize_gaussians`),
the same exactly-one-of exceptions and debug snapshot behaviour; the rasterizer returns `(color, radii, allmap)` with
allmap[9,H,W] = {expected depth sum, alpha, view-space normal (3), median depth, distortion, median weight, median
Gaussian index}.  Gradients flow from `color` and allmap channels 0-6; channels 7 and 8 (median weight and index) carry
none.  `means2D.grad` is the gradient w.r.t. a screen-space translation of each splat, in NDC units (DESIGN.md §3,
surfel rasterizer).
"""
from typing import NamedTuple

import torch

from . import _C, rasterizer
from .rasterizer import FW_MESSAGE, call_with_snapshot, check_exactly_one_of, cpu_deep_copy_tuple  # noqa: F401


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                        raster_settings):
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                     cov3Ds_precomp, raster_settings)


class _RasterizeGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                raster_settings):
        if cov3Ds_precomp is not None and cov3Ds_precomp.numel() != 0:
            raise NotImplementedError("surfel rasterizer: precomputed splat transforms (cov3D_precomp) are not supported")
        if scales.ndimension() != 2 or scales.size(1) != 2:
            raise ValueError(f"surfel rasterizer: scales must be [P,2] (two tangent scales), got {list(scales.shape)}")
        rs = raster_settings
        args = (rs.bg, means3D, colors_precomp, opacities, scales, rotations, rs.scale_modifier, rs.viewmatrix,
                rs.projmatrix, rs.tanfovx, rs.tanfovy, rs.image_height, rs.image_width, sh, rs.sh_degree, rs.campos,
                rs.prefiltered, rs.debug)
        num_rendered, color, radii, allmap, geomBuffer, binningBuffer, imgBuffer = call_with_snapshot(
            _C.rasterize_surfels, args, rs.debug, "snapshot_fw.dump", FW_MESSAGE)
        ctx.raster_settings = rs
        ctx.num_rendered = num_rendered
        ctx.save_for_backward(colors_precomp, means3D, scales, rotations, radii, sh, geomBuffer, binningBuffer,
                              imgBuffer)
        ctx.mark_non_differentiable(radii)
        return color, radii, allmap

    @staticmethod
    def backward(ctx, grad_out_color, grad_radii, grad_allmap):
        rs = ctx.raster_settings
        colors_precomp, means3D, scales, rotations, radii, sh, geomBuffer, binningBuffer, imgBuffer = ctx.saved_tensors
        args = (rs.bg, means3D, radii, colors_precomp, scales, rotations, rs.scale_modifier, rs.viewmatrix,
                rs.projmatrix, rs.tanfovx, rs.tanfovy, grad_out_color, grad_allmap, sh, rs.sh_degree, rs.campos,
                geomBuffer, ctx.num_rendered, binningBuffer, imgBuffer, rs.debug)
        (grad_means2D, grad_colors_precomp, grad_opacities, grad_means3D, grad_sh, grad_scales,
         grad_rotations) = call_with_snapshot(_C.rasterize_surfels_backward, args, rs.debug, "snapshot_bw.dump",
                                              "\nAn error occured in backward. Please forward snapshot_bw.dump for debugging.")
        return (grad_means3D, grad_means2D, grad_sh, grad_colors_precomp, grad_opacities, grad_scales, grad_rotations,
                None, None)


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool


class GaussianRasterizer(rasterizer.GaussianRasterizer):
    _function = _RasterizeGaussians

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None):
        if cov3D_precomp is not None:
            check_exactly_one_of(shs, colors_precomp, scales, rotations, cov3D_precomp)
            raise NotImplementedError("surfel rasterizer: precomputed splat transforms (cov3D_precomp) are not supported")
        return super().forward(means3D, means2D, opacities, shs, colors_precomp, scales, rotations)
