"""`vanilla_renderer`: mirrors `gaustudio/renderers/vanilla_renderer.py:7-52` (config keys of
`gaustudio/configs/vanilla.yaml:22-28`, attribute gathering, python-side SH / covariance options)."""
import torch

from . import register
from .base import BaseRenderer, eval_sh, pack_result  # noqa: F401  (eval_sh stays importable from here)


@register('vanilla_renderer')
class VanillaRenderer(BaseRenderer):
    default_conf = {
        **BaseRenderer.default_conf,
        # H100 extension (off by default = the reference's op sequence): apply exp / sigmoid / normalize /
        # cat(f_dc, f_rest) inside the projection kernel instead of as per-view torch ops (SURVEY.md §8f rank 1)
        'fused_activations': False,
    }

    def __init__(self, config) -> None:
        super().__init__(config)
        self.fused_activations = self.config['fused_activations']

    _DEFAULT_ACT = {"scale": "exp", "opacity": "sigmoid", "rot": "normalize"}

    def _can_fuse(self, m):
        if not self.fused_activations or self.convert_SHs_python or self.compute_cov3D_python:
            return False
        if not all(hasattr(m, a) for a in ("_xyz", "_scale", "_rot", "_opacity", "_f_dc", "_f_rest")):
            return False
        cfg = getattr(m, "config", None)
        if isinstance(cfg, dict) and "activations" in cfg and dict(cfg["activations"]) != self._DEFAULT_ACT:
            return False
        return m._scale.shape[-1] == 3 and m._f_rest.numel() > 0

    def render(self, viewpoint_camera, gaussian_model):
        if not self._can_fuse(gaussian_model):
            return super().render(viewpoint_camera, gaussian_model)
        from ..rasterizer import rasterize_gaussians_fused
        m = gaussian_model
        P = m._xyz.shape[0]
        screenspace = torch.zeros_like(m._xyz, requires_grad=True)
        rs = self.raster_settings(viewpoint_camera, m.active_sh_degree)
        image, radii, depth, median_map, opacity = rasterize_gaussians_fused(
            m._xyz, screenspace, m._f_dc.reshape(P, -1, 3), m._f_rest.reshape(P, -1, 3), m._opacity, m._scale, m._rot,
            rs)
        return pack_result(image, radii, depth, median_map, opacity, screenspace)

    def get_scales(self, gaussian_model):
        scales = gaussian_model.get_attribute("scale")
        if scales.shape[-1] == 2:
            scales = torch.cat([scales, torch.zeros_like(scales[:, :1]) + 1e-7], dim=-1)
        return scales
