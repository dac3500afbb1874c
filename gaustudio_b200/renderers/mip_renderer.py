"""`mip_renderer`: gaustudio's Mip-Splatting renderer (`gaustudio/renderers/mip_renderer.py`) on the Mip rasterizer of
gaustudio_b200.mip_rasterizer: the model's 3D-filtered opacities and scales, the 2D Mip filter of width `kernel_size`
in the projection.  Config keys and defaults of the reference; `bg_color` is a CPU tensor like the other renderers'
(the reference's Python list cannot be passed to the rasterizer).  `render` returns the vanilla renderer's 9-key dict."""
import math

import torch

from . import register
from .base import BaseRenderer, pack_result
from .vanilla_renderer import eval_sh


@register('mip_renderer')
class MipRenderer(BaseRenderer):
    default_conf = {
        'kernel_size': 0.3,
        'scaling_modifier': 1.,
        'white_background': False,
        'convert_SHs_python': False,
        'compute_cov3D_python': False,
        'debug': False,
    }

    def __init__(self, config) -> None:
        super().__init__()
        self.config = {**self.default_conf, **config}
        self.kernel_size = float(self.config['kernel_size'])
        if not (0.0 <= self.kernel_size < math.inf):
            raise ValueError(f"mip_renderer: kernel_size must be finite and >= 0, got {self.config['kernel_size']!r}")
        self.scaling_modifier = self.config['scaling_modifier']
        self.white_background = self.config['white_background']
        self.bg_color = torch.tensor([1, 1, 1] if self.white_background else [0, 0, 0], dtype=torch.float32)
        self.convert_SHs_python = self.config['convert_SHs_python']
        self.compute_cov3D_python = self.config['compute_cov3D_python']
        self.debug = self.config['debug']

    def get_gaussians_properties(self, viewpoint_camera, gaussian_model):
        xyz = gaussian_model.get_attribute("xyz")
        opacity = gaussian_model.get_opacity_with_3D_filter
        scales = rotations = cov3D_precomp = None
        if self.compute_cov3D_python:
            cov3D_precomp = gaussian_model.get_covariance(self.scaling_modifier)
        else:
            scales = gaussian_model.get_scaling_with_3D_filter
            rotations = gaussian_model.get_attribute("rot")
        shs = colors_precomp = None
        if self.convert_SHs_python:
            feats = gaussian_model.get_features
            shs_view = feats.transpose(1, 2).view(-1, 3, (gaussian_model.max_sh_degree + 1) ** 2)
            dir_pp = xyz - viewpoint_camera.camera_center.repeat(feats.shape[0], 1)
            sh2rgb = eval_sh(gaussian_model.active_sh_degree, shs_view, dir_pp / dir_pp.norm(dim=1, keepdim=True))
            colors_precomp = torch.clamp_min(sh2rgb + 0.5, 0.0)
        else:
            shs = gaussian_model.get_features
        return xyz, shs, colors_precomp, opacity, scales, rotations, cov3D_precomp

    def render(self, viewpoint_camera, gaussian_model):
        if getattr(gaussian_model, "filter_3D", None) is None:
            raise ValueError("mip_renderer needs a model with filter_3D: call compute_3D_filter(cameras) on a "
                             "MipPointCloud (gaustudio_b200.mip), or load a Mip-Splatting PLY with a filter_3D property")
        from ..mip_rasterizer import GaussianRasterizationSettings, GaussianRasterizer
        xyz, shs, colors_precomp, opacity, scales, rotations, cov3D_precomp = \
            self.get_gaussians_properties(viewpoint_camera, gaussian_model)
        screenspace = torch.zeros_like(xyz, requires_grad=True) + 0
        try:
            screenspace.retain_grad()
        except Exception:
            pass
        degree = gaussian_model.active_sh_degree if shs is not None else 1
        cam = viewpoint_camera
        rs = GaussianRasterizationSettings(
            image_height=int(cam.image_height), image_width=int(cam.image_width), tanfovx=math.tan(cam.FoVx * 0.5),
            tanfovy=math.tan(cam.FoVy * 0.5), kernel_size=self.kernel_size, bg=self.bg_color,
            scale_modifier=self.scaling_modifier, viewmatrix=cam.world_view_transform,
            projmatrix=cam.full_proj_transform, sh_degree=degree, campos=cam.camera_center, prefiltered=False,
            debug=self.debug)
        image, radii, depth, median_map, final_opacity = GaussianRasterizer(raster_settings=rs)(
            means3D=xyz, means2D=screenspace, opacities=opacity, shs=shs, colors_precomp=colors_precomp,
            scales=scales, rotations=rotations, cov3D_precomp=cov3D_precomp)
        return pack_result(image, radii, depth, median_map, final_opacity, screenspace)
