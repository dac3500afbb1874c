"""BaseRenderer.render: the L3 plugin call of the reference (`gaustudio/renderers/base.py:10-63`).

Contract kept: `get_gaussians_properties(camera, model)` -> (xyz, shs, colors_precomp, opacity, scales, rotations,
cov3D_precomp) with the attributes `bg_color`, `scaling_modifier`, `debug`; `render` returns the reference's 9-key
dict.  The attribute gathering of gaustudio's renderers (`vanilla_renderer.py:28-52`) lives here once: subclasses
supply only where the opacities and the scales come from, and which rasterizer and settings they render with.
Differences: no `plyfile` import (absent here, irrelevant to rendering) and the screen-space tensor lives on the
model's device instead of the literal "cuda".
"""
import math

import torch

from ..rasterizer import GaussianRasterizationSettings, GaussianRasterizer

RESULT_KEYS = ("render", "rendered_depth", "rendered_median_depth", "rendered_median_weight", "rendered_median_id",
               "viewspace_points", "visibility_filter", "rendered_final_opacity", "radii")

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


def settings_for(camera, *, bg, scale_modifier, sh_degree, debug):
    """GaussianRasterizationSettings of one view (field meaning: $RAST/.../__init__.py:160-172)."""
    return GaussianRasterizationSettings(
        image_height=int(camera.image_height), image_width=int(camera.image_width),
        tanfovx=math.tan(camera.FoVx * 0.5), tanfovy=math.tan(camera.FoVy * 0.5), bg=bg,
        scale_modifier=scale_modifier, viewmatrix=camera.world_view_transform,
        projmatrix=camera.full_proj_transform, sh_degree=sh_degree, campos=camera.camera_center,
        prefiltered=False, debug=debug)


def pack_result(image, radii, depth, median_map, opacity, screenspace):
    """The median map's three channels are (depth, weight, Gaussian id as float): forward.cu:392-394."""
    values = (image, depth, median_map[0:1], median_map[1:2], median_map[2:3].int(), screenspace, radii > 0, opacity,
              radii)
    return dict(zip(RESULT_KEYS, values))


class BaseRenderer:
    # config keys of gaustudio's renderer configs (configs/vanilla.yaml:22-28); subclasses extend or override them
    default_conf = {
        'kernel_size': 0.,
        'scaling_modifier': 1.,
        'white_background': False,
        'convert_SHs_python': False,
        'compute_cov3D_python': False,
        'debug': False,
    }
    rasterizer = GaussianRasterizer

    def __init__(self, config) -> None:
        self.config = {**self.default_conf, **config}
        self.kernel_size = self.config['kernel_size']
        self.scaling_modifier = self.config['scaling_modifier']
        self.white_background = self.config['white_background']
        # kept on the CPU like the reference (vanilla_renderer.py:23); the binding moves it (SURVEY.md §7)
        self.bg_color = torch.tensor([1, 1, 1] if self.white_background else [0, 0, 0], dtype=torch.float32)
        self.convert_SHs_python = self.config['convert_SHs_python']
        self.compute_cov3D_python = self.config['compute_cov3D_python']
        self.debug = self.config['debug']

    def get_opacity(self, gaussian_model):
        return gaussian_model.get_attribute("opacity")

    def get_scales(self, gaussian_model):
        return gaussian_model.get_attribute("scale")

    def get_gaussians_properties(self, viewpoint_camera, gaussian_model):
        xyz = gaussian_model.get_attribute("xyz")
        opacity = self.get_opacity(gaussian_model)
        scales = rotations = cov3D_precomp = None
        if self.compute_cov3D_python:
            cov3D_precomp = gaussian_model.get_covariance(self.scaling_modifier)
        else:
            scales = self.get_scales(gaussian_model)
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

    def raster_settings(self, viewpoint_camera, sh_degree):
        return settings_for(viewpoint_camera, bg=self.bg_color, scale_modifier=self.scaling_modifier,
                            sh_degree=sh_degree, debug=self.debug)

    def rasterize(self, viewpoint_camera, gaussian_model, props=None):
        """The rasterizer's outputs for one view, and the screen-space tensor its 2-D mean gradients arrive in.
        props: the 7-tuple of get_gaussians_properties when the caller has it already."""
        xyz, shs, colors_precomp, opacity, scales, rotations, cov3D_precomp = \
            props if props is not None else self.get_gaussians_properties(viewpoint_camera, gaussian_model)
        # a zero tensor in the graph: autograd hands back the 2-D (screen-space) mean gradients through it
        screenspace = torch.zeros_like(xyz, requires_grad=True) + 0
        try:
            screenspace.retain_grad()
        except Exception:
            pass
        degree = gaussian_model.active_sh_degree if shs is not None else 1
        out = self.rasterizer(raster_settings=self.raster_settings(viewpoint_camera, degree))(
            means3D=xyz, means2D=screenspace, opacities=opacity, shs=shs, colors_precomp=colors_precomp,
            scales=scales, rotations=rotations, cov3D_precomp=cov3D_precomp)
        return out, screenspace

    def render(self, viewpoint_camera, gaussian_model):
        (image, radii, depth, median_map, final_opacity), screenspace = self.rasterize(viewpoint_camera, gaussian_model)
        return pack_result(image, radii, depth, median_map, final_opacity, screenspace)
