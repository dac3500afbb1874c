"""Camera: the consumer contract the rasterizer path needs (matrices + depth->normal).

Mirrors the fields and numerics of the reference dataclass
`gaustudio/datasets/__init__.py:114-183` (`Camera._setup`), its helpers
`getWorld2View2` (`:52-64`), `getProjectionMatrix` (`:66-104`) and the
`intrinsics` / `extrinsics` properties (`:219-237`), so that
`BaseRenderer.render(camera, model)` (`gaustudio/renderers/base.py:10-63`) reads
identical `world_view_transform`, `full_proj_transform`, `camera_center`,
`FoVx`, `FoVy`, `image_width`, `image_height`.  The per-view `image`, `mask` and `depth` fields (`:139-143`) and
their resizes (`downsample`, `:246-266`) are there for the initializers that read posed views; loading them from disk
(the dataset loaders) is out of scope.
"""
import dataclasses
import math

import numpy as np
import torch


def world_to_view(R, t, translate=(0.0, 0.0, 0.0), scale=1.0):
    """W2C 4x4 (float32) from a camera-to-world rotation R and W2C translation t
    (reference: datasets/__init__.py:52-64)."""
    Rt = np.zeros((4, 4))
    Rt[:3, :3] = np.asarray(R).transpose()
    Rt[:3, 3] = np.asarray(t)
    Rt[3, 3] = 1.0
    c2w = np.linalg.inv(Rt)
    c2w[:3, 3] = (c2w[:3, 3] + np.asarray(translate)) * scale
    return np.float32(np.linalg.inv(c2w))


def projection_matrix(znear, zfar, fovX, fovY, width, height, principal_point_ndc=None):
    """OpenGL-style frustum with z_sign=+1 (reference: datasets/__init__.py:66-104)."""
    top = math.tan(fovY / 2) * znear
    bottom = -top
    right = math.tan(fovX / 2) * znear
    left = -right
    if principal_point_ndc is not None:
        focal_x = width / (2.0 * np.tan(fovX / 2.0))
        focal_y = height / (2.0 * np.tan(fovY / 2.0))
        off_x = ((width * principal_point_ndc[0] - width / 2) / focal_x) * znear
        off_y = ((height * principal_point_ndc[1] - height / 2) / focal_y) * znear
        top, bottom, left, right = top + off_y, bottom + off_y, left + off_x, right + off_x
    P = torch.zeros(4, 4)
    P[0, 0] = 2.0 * znear / (right - left)
    P[1, 1] = 2.0 * znear / (top - bottom)
    P[0, 2] = (right + left) / (right - left)
    P[1, 2] = (top + bottom) / (top - bottom)
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    return P


@dataclasses.dataclass
class Camera:
    R: np.ndarray
    T: np.ndarray
    FoVx: float
    FoVy: float
    image_width: int
    image_height: int
    znear: float = 0.1
    zfar: float = 100
    trans: np.ndarray = None
    scale: float = 1.0
    world_view_transform: torch.Tensor = None
    full_proj_transform: torch.Tensor = None
    projection_matrix: torch.Tensor = None
    camera_center: torch.Tensor = None
    principal_point_ndc: np.ndarray = None
    image: torch.Tensor = None  # [H,W,3] float in [0, 1]
    mask: torch.Tensor = None   # [H,W], nonzero = foreground
    depth: torch.Tensor = None  # [H,W] float32

    def __post_init__(self):
        self._setup()

    def _setup(self):
        if self.trans is None:
            self.trans = np.array([0.0, 0.0, 0.0])
        if self.principal_point_ndc is None:
            self.principal_point_ndc = np.array([0.5, 0.5])
        # stored transposed: flat index 4*col+row is the mathematical [row][col] (auxiliary.h:58-77)
        self.world_view_transform = torch.tensor(world_to_view(self.R, self.T, self.trans, self.scale)).transpose(0, 1)
        self.projection_matrix = projection_matrix(self.znear, self.zfar, self.FoVx, self.FoVy, self.image_width,
                                                   self.image_height, self.principal_point_ndc).transpose(0, 1)
        self.full_proj_transform = (
            self.world_view_transform.unsqueeze(0).bmm(self.projection_matrix.unsqueeze(0))).squeeze(0)
        self.camera_center = torch.inverse(self.world_view_transform)[3][:3]

    def to(self, device):
        for f in dataclasses.fields(self):
            v = getattr(self, f.name)
            if isinstance(v, torch.Tensor):
                setattr(self, f.name, v.to(device))
        return self

    @property
    def extrinsics(self):
        return self.world_view_transform.transpose(0, 1).contiguous()

    @property
    def intrinsics(self):
        fy = self.image_height / (2.0 * np.tan(self.FoVy / 2.0))
        fx = self.image_width / (2.0 * np.tan(self.FoVx / 2.0))
        return torch.tensor([[fx, 0, self.image_width * self.principal_point_ndc[0]],
                             [0, fy, self.image_height * self.principal_point_ndc[1]],
                             [0, 0, 1]]).float()

    @property
    def fx(self):
        return self.intrinsics[0, 0]

    @property
    def fy(self):
        return self.intrinsics[1, 1]

    def downsample_scale(self, scale):
        """downsample to (round(W / scale), round(H / scale)) (datasets/__init__.py:246-249)."""
        return self.downsample((round(self.image_width / scale), round(self.image_height / scale)))

    def downsample(self, resolution):
        """Resize image, mask and depth to resolution = (W, H) with PIL, as the reference does (:251-266): image and
        mask through resize_image, depth through resize_depth.  Replaces the fields (host tensors) and the size."""
        if self.image is not None:
            self.image = resize_image(self.image, resolution)[..., :3].clamp(0.0, 1.0)
        if self.mask is not None:
            self.mask = resize_image(self.mask, resolution).clamp(0.0, 1.0)
        if self.depth is not None:
            self.depth = resize_depth(self.depth, resolution)
        self.image_width, self.image_height = resolution
        return self

    def depth2point(self, depth=None, coordinate="camera"):
        """[H,W] depth (default: self.depth) -> [H,W,3] points (CUDA restatement of datasets/__init__.py:307-339)."""
        from . import ops
        if depth is None:
            depth = self.depth
        if depth is None:
            raise ValueError("Depth is not available.")
        K = self.intrinsics
        c2w = torch.inverse(self.extrinsics) if coordinate == "world" else None
        return ops.depth2point(depth, float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), c2w)

    def depth2normal(self, depth, d_min=1e-3, d_max=100000.0, coordinate="camera"):
        """[H,W] depth -> [H,W,3] normals; CUDA restatement of datasets/__init__.py:342-380 (k=3)."""
        from . import ops
        K = self.intrinsics
        rot = None
        if coordinate == "world":
            rot = self.extrinsics[:3, :3].inverse().t().contiguous().to(depth.device)
        return ops.depth2normal(depth, float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]),
                                d_min, d_max, rot)


def _host(t):
    return t.detach().cpu() if isinstance(t, torch.Tensor) else torch.from_numpy(np.asarray(t))


def resize_image(image, resolution):
    """resizeTorch (datasets/__init__.py:10-24): values scaled by 255 when the maximum is <= 1, truncated to uint8,
    resized by PIL's Image.resize with its default resample, -> float32 / 255 on the host."""
    from PIL import Image
    t = _host(image)
    if t.max() <= 1.0:
        t = t * 255.0
    pil = Image.fromarray(t.byte().numpy())
    return torch.from_numpy(np.array(pil.resize(resolution))).float() / 255.0


def resize_depth(depth, resolution):
    """resizeDepthTorch (datasets/__init__.py:26-43): PIL mode F, NEAREST -> float32 [H,W] on the host."""
    from PIL import Image
    t = _host(depth)
    if t.dim() != 2:
        raise ValueError("Input tensor must have shape [H, W]")
    pil = Image.fromarray(t.numpy().astype(np.float32))
    return torch.from_numpy(np.array(pil.resize(resolution, Image.NEAREST)).astype(np.float32))


def look_at_camera(position, target, W, H, FoVx, FoVy, up=(0.0, 0.0, 1.0), **kw):
    """Camera at `position` looking at `target` (x right, y down, z forward: the COLMAP/3DGS frame)."""
    c = np.asarray(position, dtype=np.float64)
    f = np.asarray(target, dtype=np.float64) - c
    f /= np.linalg.norm(f)
    right = np.cross(f, np.asarray(up, dtype=np.float64))
    right /= np.linalg.norm(right)
    down = np.cross(f, right)
    R = np.stack([right, down, f], axis=1)  # camera-to-world rotation (columns = camera axes)
    T = -R.T @ c
    return Camera(R=R, T=T, FoVx=FoVx, FoVy=FoVy, image_width=W, image_height=H, **kw)


def orbit_cameras(K, radius, elevation_deg, W, H, FoVx, FoVy, indices=None):
    """K cameras on a circle at `elevation_deg`, azimuth 360*k/K, looking at the origin (SURVEY.md §8d;
    same idea as gaustudio/cameras/camera_paths.py:89-102)."""
    el = math.radians(elevation_deg)
    cams = []
    for k in (range(K) if indices is None else indices):
        az = 2.0 * math.pi * k / K
        pos = (radius * math.cos(el) * math.cos(az), radius * math.cos(el) * math.sin(az), radius * math.sin(el))
        cams.append(look_at_camera(pos, (0.0, 0.0, 0.0), W, H, FoVx, FoVy))
    return cams
