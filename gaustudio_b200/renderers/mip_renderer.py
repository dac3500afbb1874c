"""`mip_renderer`: gaustudio's Mip-Splatting renderer (`gaustudio/renderers/mip_renderer.py`) on the Mip rasterizer of
gaustudio_b200.mip_rasterizer: the model's 3D-filtered opacities and scales, the 2D Mip filter of width `kernel_size`
in the projection.  Config keys and defaults of the reference; `bg_color` is a CPU tensor like the other renderers'
(the reference's Python list cannot be passed to the rasterizer).  `render` returns the vanilla renderer's 9-key dict."""
import math

from . import register
from .base import BaseRenderer
from ..mip_rasterizer import GaussianRasterizationSettings


@register('mip_renderer')
class MipRenderer(BaseRenderer):
    default_conf = {**BaseRenderer.default_conf, 'kernel_size': 0.3}

    def __init__(self, config) -> None:
        super().__init__(config)
        self.kernel_size = float(self.config['kernel_size'])
        if not (0.0 <= self.kernel_size < math.inf):
            raise ValueError(f"mip_renderer: kernel_size must be finite and >= 0, got {self.config['kernel_size']!r}")

    def get_opacity(self, gaussian_model):
        return gaussian_model.get_opacity_with_3D_filter

    def get_scales(self, gaussian_model):
        return gaussian_model.get_scaling_with_3D_filter

    def raster_settings(self, viewpoint_camera, sh_degree):
        rs = super().raster_settings(viewpoint_camera, sh_degree)
        return GaussianRasterizationSettings(kernel_size=self.kernel_size, **rs._asdict())

    def render(self, viewpoint_camera, gaussian_model):
        if getattr(gaussian_model, "filter_3D", None) is None:
            raise ValueError("mip_renderer needs a model with filter_3D: call compute_3D_filter(cameras) on a "
                             "MipPointCloud (gaustudio_b200.mip), or load a Mip-Splatting PLY with a filter_3D property")
        return super().render(viewpoint_camera, gaussian_model)
