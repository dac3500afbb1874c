"""Autograd boundary: drop-in for `gaustudio_diff_gaussian_rasterization/__init__.py` of the reference
($RAST/gaustudio_diff_gaussian_rasterization/__init__.py:21-223).

Same public names, same argument packing (19 forward / 24 backward arguments), same 5-tuple
`(color, radii, depth, median_depth[3,H,W], final_opacity)`, same saved tensors, same exceptions and the
same debug snapshot behaviour -- on top of `gaustudio_b200._C` (ctypes over the C ABI of libgsr_b200.so).
"""
from typing import NamedTuple

import torch
import torch.nn as nn

from . import _C


def cpu_deep_copy_tuple(input_tuple):
    return tuple(item.cpu().clone() if isinstance(item, torch.Tensor) else item for item in input_tuple)


def call_with_snapshot(fn, args, debug, path, message):
    """fn(*args).  With `debug`, a CPU copy of `args` taken before the call is saved to `path` if the call raises, and
    `message` is printed before the exception propagates (__init__.py:83-90)."""
    if not debug:
        return fn(*args)
    cpu_args = cpu_deep_copy_tuple(args)  # copy before they can be corrupted
    try:
        return fn(*args)
    except Exception as ex:
        torch.save(cpu_args, path)
        print(message)
        raise ex


FW_MESSAGE = "\nAn error occured in forward. Please forward snapshot_fw.dump for debugging."


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                        raster_settings):
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                     cov3Ds_precomp, raster_settings)


class _RasterizeGaussians(torch.autograd.Function):
    """Settings with a `kernel_size` field (gaustudio_b200.mip_rasterizer) select the Mip-Splatting projection, whose
    backward also needs the input opacities."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                raster_settings):
        rs = raster_settings
        mip = hasattr(rs, "kernel_size")
        args = (rs.bg, means3D, colors_precomp, opacities, scales, rotations, rs.scale_modifier, cov3Ds_precomp,
                rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, rs.image_height, rs.image_width, sh,
                rs.sh_degree, rs.campos, rs.prefiltered, rs.debug)
        if mip:
            out = call_with_snapshot(_C.rasterize_gaussians_mip, args + (rs.kernel_size,), rs.debug,
                                     "snapshot_fw.dump", FW_MESSAGE)
        else:
            out = call_with_snapshot(_C.rasterize_gaussians, args, rs.debug, "snapshot_fw.dump", FW_MESSAGE)
        num_rendered, color, depth, median_depth, final_opacity, radii, geomBuffer, binningBuffer, imgBuffer = out
        ctx.raster_settings = rs
        ctx.num_rendered = num_rendered
        saved = (colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geomBuffer, binningBuffer,
                 imgBuffer)
        if mip:
            saved += (opacities,)
        ctx.save_for_backward(*saved)
        ctx.mark_non_differentiable(radii)
        return color, radii, depth, median_depth, final_opacity

    @staticmethod
    def backward(ctx, grad_out_color, grad_radii, grad_depth, grad_median_depth, grad_final_opacity):
        rs = ctx.raster_settings
        (colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geomBuffer, binningBuffer,
         imgBuffer, *mip_opacities) = ctx.saved_tensors
        tail = (scales, rotations, rs.scale_modifier, cov3Ds_precomp, rs.viewmatrix, rs.projmatrix, rs.tanfovx,
                rs.tanfovy, grad_out_color, grad_depth, grad_median_depth, grad_final_opacity, sh, rs.sh_degree,
                rs.campos, geomBuffer, ctx.num_rendered, binningBuffer, imgBuffer, rs.debug)
        message = "\nAn error occured in backward. Writing snapshot_bw.dump for debugging.\n"
        if mip_opacities:
            args = (rs.bg, means3D, radii, colors_precomp, *mip_opacities, *tail, rs.kernel_size)
            out = call_with_snapshot(_C.rasterize_gaussians_mip_backward, args, rs.debug, "snapshot_bw.dump", message)
        else:
            args = (rs.bg, means3D, radii, colors_precomp, *tail)
            out = call_with_snapshot(_C.rasterize_gaussians_backward, args, rs.debug, "snapshot_bw.dump", message)
        (grad_means2D, grad_colors_precomp, grad_opacities, grad_means3D, grad_cov3Ds_precomp, grad_sh, grad_scales,
         grad_rotations) = out
        # order of the reference (__init__.py:146-156)
        return (grad_means3D, grad_means2D, grad_sh, grad_colors_precomp, grad_opacities, grad_scales, grad_rotations,
                grad_cov3Ds_precomp, None)


class _RasterizeGaussiansFused(torch.autograd.Function):
    """Fused-activation variant (SURVEY.md §8f rank 1): inputs are the model's RAW attributes; exp / sigmoid /
    normalize / cat(f_dc, f_rest) of `VanillaRenderer.get_gaussians_properties`
    (gaustudio/renderers/vanilla_renderer.py:28-52) happen inside the projection kernel and its backward."""

    @staticmethod
    def forward(ctx, means3D, means2D, f_dc, f_rest, opacity_logits, log_scales, raw_rotations, raster_settings):
        rs = raster_settings
        e = torch.Tensor([])
        out = _C.rasterize_gaussians(rs.bg, means3D, e, opacity_logits, log_scales, raw_rotations, rs.scale_modifier, e,
                                     rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, rs.image_height,
                                     rs.image_width, e, rs.sh_degree, rs.campos, rs.prefiltered, rs.debug,
                                     _fused=(f_dc, f_rest))
        num_rendered, color, depth, median_depth, final_opacity, radii, geomBuffer, binningBuffer, imgBuffer = out
        ctx.raster_settings, ctx.num_rendered = rs, num_rendered
        ctx.save_for_backward(means3D, f_dc, f_rest, opacity_logits, log_scales, raw_rotations, radii, geomBuffer,
                              binningBuffer, imgBuffer)
        ctx.mark_non_differentiable(radii)
        return color, radii, depth, median_depth, final_opacity

    @staticmethod
    def backward(ctx, grad_out_color, grad_radii, grad_depth, grad_median_depth, grad_final_opacity):
        rs = ctx.raster_settings
        means3D, f_dc, f_rest, opac, scales, rots, radii, geomBuffer, binningBuffer, imgBuffer = ctx.saved_tensors
        d_m2, d_op, d_m3, d_dc, d_rest, d_sc, d_rot = _C.rasterize_gaussians_fused_backward(
            rs.bg, means3D, radii, f_dc, f_rest, opac, scales, rots, rs.scale_modifier, rs.viewmatrix, rs.projmatrix,
            rs.tanfovx, rs.tanfovy, grad_out_color, grad_depth, grad_median_depth, grad_final_opacity, rs.sh_degree,
            rs.campos, geomBuffer, ctx.num_rendered, binningBuffer, imgBuffer, rs.debug)
        return d_m3, d_m2, d_dc, d_rest, d_op, d_sc, d_rot, None


def rasterize_gaussians_fused(means3D, means2D, f_dc, f_rest, opacity_logits, log_scales, raw_rotations,
                              raster_settings):
    return _RasterizeGaussiansFused.apply(means3D, means2D, f_dc, f_rest, opacity_logits, log_scales, raw_rotations,
                                          raster_settings)


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


def check_exactly_one_of(shs, colors_precomp, scales, rotations, cov3D_precomp):
    if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
        raise Exception('Please provide excatly one of either SHs or precomputed colors!')
    if ((scales is None or rotations is None) and cov3D_precomp is None) or \
            ((scales is not None or rotations is not None) and cov3D_precomp is not None):
        raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')


class GaussianRasterizer(nn.Module):
    _function = _RasterizeGaussians  # the autograd Function `forward` applies

    def __init__(self, raster_settings):
        super().__init__()
        self.raster_settings = raster_settings

    def markVisible(self, positions):
        with torch.no_grad():
            rs = self.raster_settings
            return _C.mark_visible(positions, rs.viewmatrix, rs.projmatrix)

    def visible_filter(self, means3D, scales=None, rotations=None, cov3D_precomp=None):
        """Radii [N] the Mip projection of the settings' `kernel_size` gives Gaussians at `means3D`, with nothing
        rendered: the Mip-Splatting fork's method, which Scaffold-GS uses to find the anchors in view.  Needs settings
        with a `kernel_size` (gaustudio_b200.mip_rasterizer); the radii equal those the forward would return."""
        rs = self.raster_settings
        if not hasattr(rs, "kernel_size"):
            raise TypeError("visible_filter needs rasterization settings with a kernel_size (gaustudio_b200.mip_rasterizer)")
        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
        with torch.no_grad():
            return _C.scaffold_visible(means3D, scales, rotations, cov3D_precomp, rs.scale_modifier, rs.viewmatrix,
                                       rs.projmatrix, rs.tanfovx, rs.tanfovy, rs.image_height, rs.image_width,
                                       rs.kernel_size)

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None):
        check_exactly_one_of(shs, colors_precomp, scales, rotations, cov3D_precomp)
        empty = torch.Tensor([])
        if shs is None:
            shs = empty
        if colors_precomp is None:
            colors_precomp = empty
        if scales is None:
            scales = empty
        if rotations is None:
            rotations = empty
        if cov3D_precomp is None:
            cov3D_precomp = empty
        return self._function.apply(means3D, means2D, shs, colors_precomp, opacities, scales, rotations,
                                    cov3D_precomp, self.raster_settings)
