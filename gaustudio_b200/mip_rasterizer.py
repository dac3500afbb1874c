"""Autograd boundary of the Mip-Splatting rasterizer: the public surface of the Mip-Splatting fork of
`diff_gaussian_rasterization` (what gaustudio's mip and scaffold renderers are written against), without
`subpixel_offset`.  Same 5-tuple `(color, radii, depth, median_depth[3,H,W], final_opacity)`, exceptions and debug
snapshots as `gaustudio_b200.rasterizer`; the projection applies the 2D Mip filter of width
`raster_settings.kernel_size` (include/gsr.h, gsr_forward_mip) instead of the fixed 0.3 dilation.
"""
from typing import NamedTuple

import torch
import torch.nn as nn

from . import _C
from .rasterizer import cpu_deep_copy_tuple


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                        raster_settings):
    return _RasterizeGaussiansMip.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                        cov3Ds_precomp, raster_settings)


class _RasterizeGaussiansMip(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                raster_settings):
        rs = raster_settings
        args = (rs.bg, means3D, colors_precomp, opacities, scales, rotations, rs.scale_modifier, cov3Ds_precomp,
                rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, rs.image_height, rs.image_width, sh,
                rs.sh_degree, rs.campos, rs.prefiltered, rs.debug, rs.kernel_size)
        if rs.debug:
            cpu_args = cpu_deep_copy_tuple(args)
            try:
                out = _C.rasterize_gaussians_mip(*args)
            except Exception as ex:
                torch.save(cpu_args, "snapshot_fw.dump")
                print("\nAn error occured in forward. Please forward snapshot_fw.dump for debugging.")
                raise ex
        else:
            out = _C.rasterize_gaussians_mip(*args)
        num_rendered, color, depth, median_depth, final_opacity, radii, geomBuffer, binningBuffer, imgBuffer = out
        ctx.raster_settings = rs
        ctx.num_rendered = num_rendered
        ctx.save_for_backward(colors_precomp, means3D, opacities, scales, rotations, cov3Ds_precomp, radii, sh,
                              geomBuffer, binningBuffer, imgBuffer)
        ctx.mark_non_differentiable(radii)
        return color, radii, depth, median_depth, final_opacity

    @staticmethod
    def backward(ctx, grad_out_color, grad_radii, grad_depth, grad_median_depth, grad_final_opacity):
        rs = ctx.raster_settings
        (colors_precomp, means3D, opacities, scales, rotations, cov3Ds_precomp, radii, sh, geomBuffer, binningBuffer,
         imgBuffer) = ctx.saved_tensors
        args = (rs.bg, means3D, radii, colors_precomp, opacities, scales, rotations, rs.scale_modifier, cov3Ds_precomp,
                rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, grad_out_color, grad_depth, grad_median_depth,
                grad_final_opacity, sh, rs.sh_degree, rs.campos, geomBuffer, ctx.num_rendered, binningBuffer,
                imgBuffer, rs.debug, rs.kernel_size)
        if rs.debug:
            cpu_args = cpu_deep_copy_tuple(args)
            try:
                out = _C.rasterize_gaussians_mip_backward(*args)
            except Exception as ex:
                torch.save(cpu_args, "snapshot_bw.dump")
                print("\nAn error occured in backward. Writing snapshot_bw.dump for debugging.\n")
                raise ex
        else:
            out = _C.rasterize_gaussians_mip_backward(*args)
        (grad_means2D, grad_colors_precomp, grad_opacities, grad_means3D, grad_cov3Ds_precomp, grad_sh, grad_scales,
         grad_rotations) = out
        return (grad_means3D, grad_means2D, grad_sh, grad_colors_precomp, grad_opacities, grad_scales, grad_rotations,
                grad_cov3Ds_precomp, None)


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    kernel_size: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings):
        super().__init__()
        self.raster_settings = raster_settings

    def markVisible(self, positions):
        with torch.no_grad():
            rs = self.raster_settings
            return _C.mark_visible(positions, rs.viewmatrix, rs.projmatrix)

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None):
        rs = self.raster_settings
        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception('Please provide excatly one of either SHs or precomputed colors!')
        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
        empty = torch.Tensor([])
        shs = empty if shs is None else shs
        colors_precomp = empty if colors_precomp is None else colors_precomp
        scales = empty if scales is None else scales
        rotations = empty if rotations is None else rotations
        cov3D_precomp = empty if cov3D_precomp is None else cov3D_precomp
        return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp,
                                   rs)
