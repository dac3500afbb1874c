"""Autograd boundary of the Mip-Splatting rasterizer: the public surface of the Mip-Splatting fork of
`diff_gaussian_rasterization` (what gaustudio's mip and scaffold renderers are written against), without
`subpixel_offset`.  Only the settings are its own: the rasterizer and its Function are `gaustudio_b200.rasterizer`'s,
which, given settings with a `kernel_size` field, apply the 2D Mip filter of that width (include/gsr.h,
gsr_forward_mip) instead of the fixed 0.3 dilation.  Same 5-tuple `(color, radii, depth, median_depth[3,H,W],
final_opacity)`, exceptions and debug snapshots.
"""
from typing import NamedTuple

import torch

from .rasterizer import GaussianRasterizer, cpu_deep_copy_tuple, rasterize_gaussians  # noqa: F401


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
