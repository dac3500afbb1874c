"""`vanilla_renderer`: mirrors `gaustudio/renderers/vanilla_renderer.py:7-52` (config keys of
`gaustudio/configs/vanilla.yaml:22-28`, attribute gathering, python-side SH / covariance options)."""
import torch

from . import register
from .base import BaseRenderer

C0 = 0.28209479177387814
C1 = 0.4886025119029199
C2 = [1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396]
C3 = [-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
      1.445305721320277, -0.5900435899266435]


def eval_sh(deg, sh, dirs):
    """Real SH evaluation, sh[..., C, (deg+1)^2], dirs[..., 3] (same basis as gaustudio/utils/sh_utils.py:57-112)."""
    result = C0 * sh[..., 0]
    if deg > 0:
        x, y, z = dirs[..., 0:1], dirs[..., 1:2], dirs[..., 2:3]
        result = result - C1 * y * sh[..., 1] + C1 * z * sh[..., 2] - C1 * x * sh[..., 3]
        if deg > 1:
            xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
            result = (result + C2[0] * xy * sh[..., 4] + C2[1] * yz * sh[..., 5] +
                      C2[2] * (2.0 * zz - xx - yy) * sh[..., 6] + C2[3] * xz * sh[..., 7] +
                      C2[4] * (xx - yy) * sh[..., 8])
            if deg > 2:
                result = (result + C3[0] * y * (3 * xx - yy) * sh[..., 9] + C3[1] * xy * z * sh[..., 10] +
                          C3[2] * y * (4 * zz - xx - yy) * sh[..., 11] +
                          C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * sh[..., 12] +
                          C3[4] * x * (4 * zz - xx - yy) * sh[..., 13] + C3[5] * z * (xx - yy) * sh[..., 14] +
                          C3[6] * x * (xx - 3 * yy) * sh[..., 15])
    return result


@register('vanilla_renderer')
class VanillaRenderer(BaseRenderer):
    default_conf = {
        'kernel_size': 0.,
        'scaling_modifier': 1.,
        'white_background': False,
        'convert_SHs_python': False,
        'compute_cov3D_python': False,
        'debug': False,
        # H100 extension (off by default = the reference's op sequence): apply exp / sigmoid / normalize /
        # cat(f_dc, f_rest) inside the projection kernel instead of as per-view torch ops (SURVEY.md §8f rank 1)
        'fused_activations': False,
    }

    def __init__(self, config) -> None:
        super().__init__()
        self.config = {**self.default_conf, **config}
        self.kernel_size = self.config['kernel_size']
        self.scaling_modifier = self.config['scaling_modifier']
        self.white_background = self.config['white_background']
        # kept on the CPU like the reference (vanilla_renderer.py:23); the binding moves it (SURVEY.md §7)
        self.bg_color = torch.tensor([1, 1, 1] if self.white_background else [0, 0, 0], dtype=torch.float32)
        self.convert_SHs_python = self.config['convert_SHs_python']
        self.compute_cov3D_python = self.config['compute_cov3D_python']
        self.debug = self.config['debug']
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
        from .base import pack_result, settings_for
        m = gaussian_model
        P = m._xyz.shape[0]
        screenspace = torch.zeros_like(m._xyz, requires_grad=True)
        rs = settings_for(viewpoint_camera, bg=self.bg_color, scale_modifier=self.scaling_modifier,
                          sh_degree=m.active_sh_degree, debug=self.debug)
        image, radii, depth, median_map, opacity = rasterize_gaussians_fused(
            m._xyz, screenspace, m._f_dc.reshape(P, -1, 3), m._f_rest.reshape(P, -1, 3), m._opacity, m._scale, m._rot,
            rs)
        return pack_result(image, radii, depth, median_map, opacity, screenspace)

    def get_gaussians_properties(self, viewpoint_camera, gaussian_model):
        xyz = gaussian_model.get_attribute("xyz")
        opacity = gaussian_model.get_attribute("opacity")
        scales = rotations = cov3D_precomp = None
        if self.compute_cov3D_python:
            cov3D_precomp = gaussian_model.get_covariance(self.scaling_modifier)
        else:
            scales = gaussian_model.get_attribute("scale")
            if scales.shape[-1] == 2:
                scales = torch.cat([scales, torch.zeros_like(scales[:, :1]) + 1e-7], dim=-1)
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
