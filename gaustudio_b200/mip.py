"""MipPointCloud: the Gaussian container of Mip-Splatting (gaustudio's `mip_pcd` model, `models/mip_sg.py`).

A GaussianPointCloud plus `filter_3D` [P,1], the per-Gaussian 3D smoothing filter: the world-space size of one pixel at
the Gaussian's nearest depth over the training cameras, times sqrt(0.2).  It carries no gradient and is recomputed by
`compute_3D_filter` (one CUDA pass over all cameras, gsr_mip_filter3d) rather than trained.  The filtered attributes
fold it into the scales and opacities:

    get_scaling_with_3D_filter = sqrt(s^2 + f^2)
    get_opacity_with_3D_filter = sigmoid(o) * sqrt(prod(s^2) / prod(s^2 + f^2))

`get_covariance` is built from the FILTERED scales.  The reference model builds it from the raw scales, so there its
`compute_cov3D_python` option renders a different picture from the default; here both options agree.
"""
import torch
import torch.nn.functional as F

from .synthetic import GaussianPointCloud


class MipPointCloud(GaussianPointCloud):
    def __init__(self, xyz, scale, rot, opacity, f_dc, f_rest, sh_degree=3, active_sh_degree=None, filter_3D=None):
        super().__init__(xyz, scale, rot, opacity, f_dc, f_rest, sh_degree, active_sh_degree)
        self.filter_3D = None if filter_3D is None else filter_3D.detach().reshape(-1, 1)

    @classmethod
    def from_model(cls, model, filter_3D=None):
        """A MipPointCloud sharing the raw attribute tensors of `model` (a GaussianPointCloud)."""
        return cls(model._xyz, model._scale, model._rot, model._opacity, model._f_dc, model._f_rest,
                   model.max_sh_degree, model.active_sh_degree, filter_3D)

    def to(self, device):
        super().to(device)
        if self.filter_3D is not None:
            self.filter_3D = self.filter_3D.to(device)
        return self

    def _filter(self):
        if self.filter_3D is None:
            raise RuntimeError("MipPointCloud has no filter_3D: call compute_3D_filter(cameras) first, or load a "
                               "Mip-Splatting PLY that has a filter_3D property")
        return self.filter_3D

    @torch.no_grad()
    def compute_3D_filter(self, cameras):
        """filter_3D from the training cameras (Camera objects, e.g. io.load_cameras_json) in one CUDA pass.
        Raises ValueError when no camera sees any Gaussian."""
        from . import _C
        self.filter_3D = _C.mip_filter3d(self._xyz.detach(), cameras).reshape(-1, 1)
        return self.filter_3D

    @property
    def get_scaling_with_3D_filter(self):
        s = self.get_attribute("scale")
        return torch.sqrt(torch.square(s) + torch.square(self._filter()))

    @property
    def get_opacity_with_3D_filter(self):
        s2 = torch.square(self.get_attribute("scale"))
        det1 = s2[:, 0] * s2[:, 1] * s2[:, 2]
        s2f = s2 + torch.square(self._filter())
        det2 = s2f[:, 0] * s2f[:, 1] * s2f[:, 2]
        return self.get_attribute("opacity") * torch.sqrt(det1 / det2)[..., None]

    def get_covariance(self, scaling_modifier=1):
        """Packed 3D covariance [P,6] (xx, xy, xz, yy, yz, zz) of the filtered scales and the normalised rotations."""
        s = scaling_modifier * self.get_scaling_with_3D_filter
        r, x, y, z = F.normalize(self._rot).unbind(1)
        R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                         2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                         2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)
        L = R * s[:, None, :]
        S = L @ L.transpose(1, 2)
        return torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], 1)
