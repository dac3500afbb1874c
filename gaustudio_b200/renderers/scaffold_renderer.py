"""`scaffold_renderer`: gaustudio's Scaffold-GS renderer (`gaustudio/renderers/scaffold_renderer.py`) on the Mip
rasterizer of gaustudio_b200.mip_rasterizer.  Per view: anchor visibility (`visible_filter`, one CUDA pass), the anchor
MLPs in torch, the neural-Gaussian decoding in CUDA (gaustudio_b200.scaffold.decode), then the Mip forward with
`colors_precomp`.  Config keys and defaults of the reference; `convert_SHs_python` and `compute_cov3D_python` are
accepted and unused (the neural Gaussians have no SH and their covariance comes from the decoded scales), `bg_color` is
a CPU tensor like the other renderers'.  `render` returns the vanilla renderer's 9-key dict plus what Scaffold-GS
training reads for anchor growing: `visible_mask` [N], `selection_mask` [Nv*k], `neural_opacity` [Nv*k,1] and
`scaling` [M,3]."""
import math

import torch

from . import register
from .base import BaseRenderer, pack_result
from .. import scaffold
from ..mip_rasterizer import GaussianRasterizationSettings


@register('scaffold_renderer')
class ScaffoldRenderer(BaseRenderer):
    def __init__(self, config) -> None:
        super().__init__(config)
        self.kernel_size = float(self.config['kernel_size'])
        if not (0.0 <= self.kernel_size < math.inf):
            raise ValueError(f"scaffold_renderer: kernel_size must be finite and >= 0, got {self.config['kernel_size']!r}")

    def raster_settings(self, viewpoint_camera, sh_degree):
        rs = super().raster_settings(viewpoint_camera, sh_degree)
        return GaussianRasterizationSettings(kernel_size=self.kernel_size, **rs._asdict())

    def prefilter_voxel(self, viewpoint_camera, gaussian_model):
        """Anchors whose Gaussian (the first three scales, the anchor's rotation) has a radius in this view."""
        rasterizer = self.rasterizer(raster_settings=self.raster_settings(viewpoint_camera, 1))
        radii = rasterizer.visible_filter(means3D=gaussian_model.get_attribute("anchor"),
                                          scales=gaussian_model.get_attribute("scale")[:, :3],
                                          rotations=gaussian_model.get_attribute("rot"))
        return radii > 0

    def neural_gaussians(self, viewpoint_camera, gaussian_model):
        """-> (xyz, rgb, opacity, scales, rotations) of the kept neural Gaussians, and the training extras."""
        visible_mask = self.prefilter_voxel(viewpoint_camera, gaussian_model)
        vis = visible_mask.nonzero().flatten()
        opacity, color, cov = scaffold.mlp_outputs(gaussian_model, vis, viewpoint_camera.camera_center)
        gaussians = scaffold.decode(gaussian_model.get_attribute("anchor"), gaussian_model.get_attribute("offset"),
                                    gaussian_model.get_attribute("scale"), opacity, color, cov, vis)
        neural_opacity = opacity.reshape(-1, 1)
        extras = dict(visible_mask=visible_mask, selection_mask=neural_opacity.view(-1) > 0.0,
                      neural_opacity=neural_opacity, scaling=gaussians[3])
        return gaussians, extras

    def get_gaussians_properties(self, viewpoint_camera, gaussian_model):
        (xyz, rgb, opacity, scales, rotations), _ = self.neural_gaussians(viewpoint_camera, gaussian_model)
        return xyz, None, rgb, opacity, scales, rotations, None

    def render(self, viewpoint_camera, gaussian_model, subpixel_offset=None):
        if subpixel_offset is not None:
            raise NotImplementedError("scaffold_renderer: subpixel_offset is not supported (pixel centres only)")
        (xyz, rgb, opacity, scales, rotations), extras = self.neural_gaussians(viewpoint_camera, gaussian_model)
        props = (xyz, None, rgb, opacity, scales, rotations, None)
        (image, radii, depth, median_map, final_opacity), screenspace = \
            self.rasterize(viewpoint_camera, gaussian_model, props)
        return {**pack_result(image, radii, depth, median_map, final_opacity, screenspace), **extras}
