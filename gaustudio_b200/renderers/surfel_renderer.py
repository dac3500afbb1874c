"""`surfel_renderer`: the 2DGS renderer of gaustudio (`gaustudio/renderers/surfel_renderer.py`, selected by
`configs/2dgs.yaml`) on the surfel rasterizer of csrc/gsr_surfel.cu.  Config keys of 2dgs.yaml plus `kernel_size`
(accepted, unused).  `render` returns the reference's dict; `rendered_normal` is in world space."""
import torch

from . import register
from .base import BaseRenderer
from ..surfel_rasterizer import GaussianRasterizer


@register('surfel_renderer')
class SurfelRenderer(BaseRenderer):
    rasterizer = GaussianRasterizer

    def render(self, viewpoint_camera, gaussian_model):
        (image, radii, allmap), screenspace = self.rasterize(viewpoint_camera, gaussian_model)
        alpha = allmap[1:2]
        normal = (allmap[2:5].permute(1, 2, 0) @ viewpoint_camera.world_view_transform[:3, :3].T).permute(2, 0, 1)
        median = torch.nan_to_num(allmap[5:6], 0, 0)
        depth = torch.nan_to_num(allmap[0:1] / alpha, 0, 0)
        return {"render": image,
                "rendered_normal": normal,
                "rendered_depth": depth,
                "rendered_median_depth": median,
                "rendered_median_weight": allmap[7:8],
                "rendered_median_id": allmap[8:9].int(),
                "viewspace_points": screenspace,
                "visibility_filter": radii > 0,
                "rendered_final_opacity": alpha,
                "radii": radii}
