"""Gaussian initialization on the GPU: the initializers of gaustudio/pipelines/initializers/ that need no external
tool, behind the reference's registry surface (`initializers/__init__.py:10-24`).

  dist2(xyz)                         distCUDA2 of simple_knn: mean squared distance to the 3 nearest other points
  normal2rotation(normals)           pcd.py:12-37 (the raw quaternion of [R0 | R1 | n])
  make({"name": "pcd", "model_path": ...})           pcd.py:39-77
  make({"name": "mesh", "n_gaussians_per_surface_triangle": n})   mesh.py:74-250 (SuGaR placement)
  make({"name": "voxel", "voxel_size": s})           mesh.py:252-442
  make({"name": "VisualHull", "resolution": 128, ...})   mask.py:16-108 (space carving against the views' masks)
  make({"name": "depth", "workspace_dir": ...})        depth.py:18-91 (back-projected depth maps)

An initializer is called as the reference calls it: `init(model, mesh=None, dataset=None, overwrite=False)` for the
mesh-based ones, `init(model, dataset, overwrite=False)` for VisualHull and depth, whose dataset is an iterable of
cameras carrying masks or depth maps.  It fills `model` (a GaussianPointCloud) through `create_from_attribute` and
returns it.  The kernels are in csrc/gsr_init.cu, csrc/gsr_clean.cu (MODE_DIST2) and csrc/gsr_hull.cu; DESIGN.md 7j
and 7k state the contracts and the departures from the reference.
"""
from collections.abc import Mapping
import copy
import ctypes as C
import math
import os
import tempfile

import numpy as np
import torch

from . import _lib
from ._lib import ALLOC, call, ptr

initializers = {}  # name -> class (public, like the reference's module-level dict)


def register(name):
    def _add(cls):
        initializers[name] = cls
        return cls
    return _add


def make(config):
    """`config`: a registered name, or a mapping with `name` (the mapping itself is handed to the constructor)."""
    if isinstance(config, str):
        name, options = config, {}
    elif isinstance(config, Mapping) or hasattr(config, "get"):
        name, options = config.get("name"), config
    else:
        raise ValueError("Initializer name is required")
    if not name:
        raise ValueError("Initializer name is required")
    try:
        cls = initializers[name]
    except KeyError:
        raise ValueError(f"Unknown initializer: {name}") from None
    return cls(options)


_SCRATCH = 1  # slots of _lib.scratch
_VOX_COLUMNS, _VOX_HITS, _VOX_SORT, _VOX_OUT = 2, 3, 4, 5


def _points(t, name, dtype=torch.float32):
    if not isinstance(t, torch.Tensor):
        raise ValueError(f"{name} must be a tensor")
    if t.dtype != dtype:
        raise ValueError(f"{name} must be {dtype}, got {t.dtype}")
    if t.dim() != 2 or t.shape[1] != 3:
        raise ValueError(f"{name} must be [N,3], got {tuple(t.shape)}")
    if t.shape[0] > 2**31 - 1:
        raise ValueError(f"{name} holds more than 2^31-1 rows")


def dist2(xyz):
    """distCUDA2(xyz): xyz [P,3] float32 CUDA -> [P] float32, for each point the mean of the squared distances to its
    3 nearest other points (exact, in double, rounded once; duplicates count at 0; a missing neighbour, P <= 3,
    counts as +inf).  Non-finite xyz raises ValueError after the search has run (one read-back)."""
    _points(xyz, "xyz")
    if not xyz.is_cuda:
        raise ValueError("xyz must be a CUDA tensor (dist2 has no CPU path)")
    x, dev, n = xyz.detach().contiguous(), xyz.device, xyz.shape[0]
    out = torch.empty(n, dtype=torch.float32, device=dev)
    if n == 0:
        return out
    with _lib.scratch(dev):
        call("gsr_dist2", dev, n, ptr(x), ALLOC, _SCRATCH, ptr(out))
    if not bool(torch.isfinite(x).all()):
        raise ValueError("xyz must be finite")
    return out


def normal2rotation(normals):
    """normal2rotation of pcd.py:12-37 on normals [N,3] float32 CUDA -> [N,4] float32, the raw quaternion
    (rotmat2quaternion with the + 1e-6 trace, not normalised).  A normal with n_z = 0 has R1 = 0 (torch.sign(0) = 0);
    an all-zero normal gives (sqrt(2 + 1e-6) / 2, 0, 0, 0)."""
    _points(normals, "normals")
    if not normals.is_cuda:
        raise ValueError("normals must be a CUDA tensor")
    n = normals.detach().contiguous()
    rot = torch.empty(n.shape[0], 4, dtype=torch.float32, device=n.device)
    if n.shape[0]:
        call("gsr_normal2rotation", n.device, n.shape[0], ptr(n), ptr(rot))
    return rot


def _numpy_inverse_sigmoid(x):
    return np.log(x / (1 - x))


class BaseInitializer:
    """gaustudio/pipelines/initializers/base.py: `init(model, mesh=None, dataset=None, overwrite=False)`."""

    def __init__(self, config):
        self.initializer_config = config if config is not None else {}

    def __call__(self, model, mesh=None, dataset=None, overwrite=False):
        return self.build_model(model, mesh)


@register("pcd")
class PcdInitializer(BaseInitializer):
    """pcd.py:39-77: the point cloud at `model_path` (a PLY with x y z [nx ny nz] [red green blue]): colours
    uchar / 255 as open3d reads them, rotations normal2rotation(normals) when the file has normals, the scale from
    dist2 and opacity inverse_sigmoid(0.1) in float64."""

    def __init__(self, config):
        super().__init__(config)
        self.model_path = self.initializer_config.get("model_path", None)

    def build_model(self, model, mesh=None):
        from .io import read_ply_vertices
        if _device_of(model).type != "cuda":
            raise ValueError("the pcd initializer sets scales with dist2, which has no CPU path: use a CUDA model")
        if self.model_path is None or not os.path.exists(self.model_path):
            raise FileNotFoundError(f"PCD file not found: {self.model_path}")
        v = read_ply_vertices(self.model_path)
        names = v.dtype.names
        points = np.stack([v[k] for k in "xyz"], axis=1).astype(np.float64)
        colors = normals = None
        if all(k in names for k in ("red", "green", "blue")):
            c = np.stack([v[k] for k in ("red", "green", "blue")], axis=1)
            colors = c.astype(np.float64) / 255.0 if c.dtype == np.uint8 else c.astype(np.float64)
        if all(k in names for k in ("nx", "ny", "nz")):
            normals = np.stack([v[k] for k in ("nx", "ny", "nz")], axis=1).astype(np.float64)
        dev = _device_of(model)
        rot = None
        if normals is not None and len(normals):
            rot = normal2rotation(torch.from_numpy(normals).float().to(dev))
        elif normals is not None:
            rot = torch.empty(0, 4)
        opacity = _numpy_inverse_sigmoid(0.1 * np.ones((points.shape[0], 1)))
        model.create_from_attribute(xyz=torch.from_numpy(points).float(), rgb=colors, scale=None, opacity=opacity,
                                    rot=rot)
        return model


def _device_of(model):
    return model._xyz.device if getattr(model, "_xyz", None) is not None else torch.device("cuda")


def _mesh_arrays(mesh, dev):
    """(vertices [V,3] float32, faces [F,3] int64, colors [V,3] float32 | None) on dev from a tuple or a PLY path;
    shapes, dtypes and face indices are checked before any kernel runs."""
    if isinstance(mesh, (str, os.PathLike)):
        from .io import load_mesh_ply
        mesh = load_mesh_ply(mesh)
    if not isinstance(mesh, (tuple, list)) or len(mesh) != 3:
        raise ValueError("mesh must be (vertices, faces, colors | None) or a path to a mesh PLY")
    v, f, c = mesh
    _points(v, "vertices")
    if not isinstance(f, torch.Tensor) or f.dtype != torch.int64 or f.dim() != 2 or f.shape[1] != 3:
        raise ValueError("faces must be an int64 tensor [F,3]")
    if c is not None:
        _points(c, "colors")
        if c.shape != v.shape:
            raise ValueError("colors must have one row per vertex")
    if v.shape[0] == 0 or f.shape[0] == 0:
        raise ValueError("the mesh has no vertices or no faces")
    if f.shape[0] > (2**31 - 1) // 6:
        raise ValueError("the mesh has too many faces")
    if dev.type != "cuda":
        raise ValueError("mesh initialization has no CPU path: the model must be on a CUDA device")
    v, f = v.detach().to(dev).contiguous(), f.detach().to(dev).contiguous()
    c = None if c is None else c.detach().to(dev).contiguous()
    lo, hi, finite = torch.stack([f.min(), f.max(), torch.isfinite(v).all().long()]).tolist()
    if lo < 0 or hi >= v.shape[0]:
        raise ValueError("face indices must lie in [0, V)")
    if not finite:
        raise ValueError("vertices must be finite")
    return v, f, c


def vertex_normals(vertices, faces):
    """open3d's compute_vertex_normals on CUDA tensors: the sum of the unnormalised face normals of each vertex in
    ascending face order, in double, normalised (a zero sum stays zero), rounded to float32.  Not mesh.vertex_normals
    (pytorch3d's, for render_mesh)."""
    dev = vertices.device
    out = torch.empty_like(vertices)
    with _lib.scratch(dev):
        call("gsr_mesh_vertex_normals", dev, vertices.shape[0], ptr(vertices), faces.shape[0], ptr(faces), ALLOC,
             _SCRATCH, ptr(out))
    return out


_N_SLOTS = (1, 3, 4, 6)


@register("mesh")
class MeshInitializer(BaseInitializer):
    """mesh.py:74-250, SuGaR's placement: n Gaussians per face (the config key `n_gaussians_per_surface_triangle`,
    1, 3, 4 or 6, default 1; the reference never reads the key), rows face-major and slot-minor."""

    def __init__(self, config):
        super().__init__(config)
        n = self.initializer_config.get("n_gaussians_per_surface_triangle", 1)
        if isinstance(n, bool) or not isinstance(n, (int, np.integer)) or int(n) not in _N_SLOTS:
            raise ValueError(f"n_gaussians_per_surface_triangle must be 1, 3, 4 or 6, got {n!r}")
        self.n_gaussians_per_surface_triangle = int(n)

    def build_model(self, model, mesh=None):
        dev = _device_of(model)
        v, f, c = _mesh_arrays(mesh, dev)
        n, F = self.n_gaussians_per_surface_triangle, f.shape[0]
        vn = vertex_normals(v, f)
        P = F * n
        xyz = torch.empty(P, 3, device=dev)
        rot = torch.empty(P, 4, device=dev)
        f_dc = torch.empty(P, 1, 3, device=dev)
        scale = torch.empty(P, 3, device=dev)
        opacity = torch.empty(P, 1, device=dev)
        call("gsr_mesh_gaussians", dev, F, n, ptr(v), ptr(f), ptr(vn), ptr(c), ptr(xyz), ptr(rot), ptr(f_dc),
             ptr(scale), ptr(opacity))
        # what create_from_attribute would store from the kernel's (xyz, rgb, scale, rot, opacity); the kernel forms
        # RGB2SH itself, so its f_dc goes in directly
        model._set_attributes(xyz, f_dc, scale, rot, opacity)
        return model


@register("voxel")
class VoxelInitializer(BaseInitializer):
    """mesh.py:252-442: the mesh normalised into [-0.5, 0.5]^3, voxelised at `voxel_size` (the config key, default
    1/256; int(round(1 / voxel_size)) cells per axis, 1..1024), one Gaussian per occupied voxel at its centre mapped
    back, scale voxel_size * extent * 0.8, opacity logit +inf, rotation normalize(randn(4)) from `generator`.  Colour:
    the barycentric colour of the closest point of the mesh (the reference's call does not exist in open3d, so it
    paints every voxel grey); a mesh without colours gives white."""

    def __init__(self, config):
        super().__init__(config)
        vs = self.initializer_config.get("voxel_size", 1 / 256)
        if isinstance(vs, bool) or not isinstance(vs, (int, float, np.integer, np.floating)) or \
                not (math.isfinite(vs) and vs > 0) or not 1 <= int(round(1 / vs)) <= 1024:
            raise ValueError(f"voxel_size must be positive with round(1 / voxel_size) in 1..1024, got {vs!r}")
        self.voxel_size = float(vs)
        self.res = int(round(1 / self.voxel_size))

    def __call__(self, model, mesh=None, dataset=None, overwrite=False, generator=None):
        return self.build_model(model, mesh, generator)

    def build_model(self, model, mesh=None, generator=None):
        dev = _device_of(model)
        v, f, c = _mesh_arrays(mesh, dev)
        vn, center, scale = normalize_mesh(v)
        cells32, offsets, tris = voxelize(vn, f, self.res, self.voxel_size)
        U = cells32.shape[0]
        if U == 0:
            raise ValueError("No voxels generated from mesh")
        cells = cells32.long()
        ijk = torch.stack([cells // (self.res * self.res), cells // self.res % self.res, cells % self.res], 1)
        centers = (ijk.double() + 0.5) * self.voxel_size + -0.5  # open3d's GetVoxelCenterCoordinate
        points = (centers * scale + center).float()
        rgb = None
        if c is not None:
            rgb = torch.empty(U, 3, device=dev)
            call("gsr_voxel_colors", dev, U, ptr(cells32), ptr(offsets), ptr(tris), self.res, self.voxel_size, ptr(vn),
                 ptr(f), ptr(c), ptr(rgb))
        voxel_scale = self.voxel_size * float(scale) * 0.8
        scales = torch.log(torch.full((U, 3), voxel_scale, device=dev) + 1e-7)
        opacity = torch.full((U, 1), math.inf, device=dev)
        rot = torch.nn.functional.normalize(torch.randn(U, 4, generator=generator), dim=-1)
        model.create_from_attribute(xyz=points, rgb=rgb, scale=scales, opacity=opacity, rot=rot)
        return model


def normalize_mesh(vertices):
    """mesh.py:325-350 in double: (v - centre) / scale clipped to +-(0.5 - 1e-6), centre the AABB midpoint and scale
    its largest extent.  -> (normalised vertices [V,3] float64, centre [3] float64, scale 0-dim float64)."""
    v = vertices.double()
    lo, hi = v.min(0).values, v.max(0).values
    center = (lo + hi) / 2
    scale = (hi - lo).max()
    return ((v - center) / scale).clamp(-0.5 + 1e-6, 0.5 - 1e-6).contiguous(), center, scale


def voxelize(vertices, faces, res, voxel_size):
    """open3d's VoxelGrid::CreateFromTriangleMeshWithinBounds on [-0.5, 0.5]^3: vertices [V,3] float64 and faces
    [F,3] int64 CUDA -> (cells int32 [U] ascending linear indices (i res + j) res + k of the occupied cells, offsets
    int32 [U+1], triangles int32 [H]: cell u holds triangles[offsets[u]:offsets[u+1]], ascending)."""
    dev = vertices.device
    npairs = C.c_int64(0)
    with _lib.scratch(dev) as bufs:
        U = call("gsr_voxelize", dev, vertices.shape[0], ptr(vertices), faces.shape[0], ptr(faces), int(res),
                 float(voxel_size), ALLOC, _VOX_COLUMNS, _VOX_HITS, _VOX_SORT, _VOX_OUT, C.byref(npairs))
    H = npairs.value
    if U == 0:
        return (torch.empty(0, dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int32, device=dev),
                torch.empty(0, dtype=torch.int32, device=dev))
    out = bufs[_VOX_OUT].view(torch.int32)
    return out[:U], out[U:2 * U + 1], out[2 * U + 1:2 * U + 1 + H]


# ---- VisualHull (mask.py) and depth (depth.py): initializers that read posed views (csrc/gsr_hull.cu, DESIGN.md 7k) --
MAX_HULL_RES = 512  # the marching cubes' limit


def _workspace(config):
    ws = config.get("workspace_dir")
    if ws is None:
        ws = tempfile.mkdtemp()
    os.makedirs(ws, exist_ok=True)
    return ws


def scene_extent(dataset, cameras):
    """-> (translate [3] float64, min_extent): the dataset's `cameras_center` / `cameras_min_extent` when it has them,
    else getNerfppNorm's `translate` / `min_radius` of the cameras (the values the reference's loaders store there)."""
    if hasattr(dataset, "cameras_center") and hasattr(dataset, "cameras_min_extent"):
        t = dataset.cameras_center
        t = t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else t
        return np.asarray(t, np.float64).reshape(3), float(dataset.cameras_min_extent)
    from .extract import getNerfppNorm
    norm = getNerfppNorm(cameras)
    return np.asarray(norm["translate"], np.float64).reshape(3), float(norm["min_radius"])


def _check_views(cameras):
    for cam in cameras:
        W, H = int(cam.image_width), int(cam.image_height)
        if W < 1 or H < 1:
            raise ValueError(f"camera size must be positive, got {W}x{H}")
        m = getattr(cam, "mask", None)
        if m is not None and tuple(m.shape) != (H, W):
            raise ValueError(f"a mask must have the camera's shape [H,W] = [{H},{W}], got {list(m.shape)}")


def _hull_views(cameras, dev):
    """Camera records of gsr_hull_carve on dev: (proj float32 [C,16], views int64 [C,3], masks uint8 [sum H W])."""
    proj, views, masks, off = [], [], [], 0
    for cam in cameras:
        W, H = int(cam.image_width), int(cam.image_height)
        m = getattr(cam, "mask", None)
        if m is not None:
            masks.append(m)
        views.append((W, H, off if m is not None else -1))
        off += H * W if m is not None else 0
        proj.append(torch.as_tensor(cam.full_proj_transform).detach().float().cpu().reshape(16))
    P = torch.stack(proj).to(dev) if proj else torch.empty(0, 16, device=dev)
    V = torch.tensor(views, dtype=torch.int64).reshape(-1, 3).to(dev)
    M = torch.cat([(torch.as_tensor(m).to(dev) != 0).to(torch.uint8).reshape(-1) for m in masks]) if masks else None
    return P.contiguous(), V.contiguous(), M


def _hull_args(res, radius, translate):
    if isinstance(res, bool) or not isinstance(res, (int, np.integer)) or not 2 <= int(res) <= MAX_HULL_RES:
        raise ValueError(f"resolution must be an integer in 2..{MAX_HULL_RES}, got {res!r}")
    if not (math.isfinite(radius) and radius > 0):
        raise ValueError(f"the carving radius must be positive and finite, got {radius!r} (one camera, or cameras "
                         "at one point, give 0)")
    t = np.asarray(translate, np.float64).reshape(3)
    if not np.isfinite(t).all():
        raise ValueError("translate must be finite")
    return int(res), float(radius), t


def visual_hull_carve(cameras, res, radius, translate, device="cuda"):
    """The carving of mask.py:38-69: occupancy uint8 [res,res,res] (the reference's `volume`) of the nodes
    np.meshgrid(lin, lin, lin) - translate, lin = np.linspace(-radius, radius, res), that pass every camera's
    insideView against its mask (no mask: the view frustum alone).  One kernel; DESIGN.md 7k."""
    res, radius, t = _hull_args(res, radius, translate)
    cameras = list(cameras)
    _check_views(cameras)
    dev = torch.device(device)
    if dev.type != "cuda":
        raise ValueError("the visual hull has no CPU path: use a CUDA device")
    P, V, M = _hull_views(cameras, dev)
    occ = torch.empty(res, res, res, dtype=torch.uint8, device=dev)
    call("gsr_hull_carve", dev, res, radius, *map(float, t), len(cameras), ptr(P), ptr(V), ptr(M), ptr(occ))
    return occ


def visual_hull_mesh(occ, threshold, radius, translate):
    """extract_mesh of mask.py:82-93 on a carved occupancy: marching cubes at `threshold`, vertices mapped to the world
    -> (vertices [V,3] float32, faces [F,3] int64) on occ's device, faces facing the carved side."""
    if not (isinstance(occ, torch.Tensor) and occ.is_cuda and occ.dtype == torch.uint8 and occ.dim() == 3
            and occ.shape[0] == occ.shape[1] == occ.shape[2]):
        raise ValueError("occ must be a cubic uint8 CUDA tensor [res,res,res]")
    res, radius, t = _hull_args(occ.shape[0], radius, translate)
    if not 0.0 < threshold < 1.0:
        raise ValueError(f"threshold must be in (0, 1), got {threshold!r}")
    dev, occ = occ.device, occ.contiguous()
    return _lib.call_mesh("gsr_hull_marching_cubes", dev, res, ptr(occ), float(threshold), radius, *map(float, t))


@register("VisualHull")
class VisualHullInitializer(BaseInitializer):
    """mask.py:16-108: carve a `resolution`^3 grid of half-width r = cameras_min_extent * radius_scale around the
    scene centre against every camera's mask, mesh the occupancy at `threshold` into `workspace_dir`/visual_hull.ply,
    and put one Gaussian on each mesh vertex with the reference's constants: rgb 0.5, opacity logit 0.1, log-scale 0.01
    (passed to create_from_attribute unchanged).  Returns the model (the reference returns None)."""

    def __init__(self, config):
        super().__init__(config)
        cfg = self.initializer_config
        res, th, rs = cfg.get("resolution", 128), cfg.get("threshold", 0.5), cfg.get("radius_scale", 1.2)
        if isinstance(res, bool) or not isinstance(res, (int, np.integer)) or not 2 <= int(res) <= MAX_HULL_RES:
            raise ValueError(f"resolution must be an integer in 2..{MAX_HULL_RES}, got {res!r}")
        if isinstance(th, bool) or not isinstance(th, (int, float, np.integer, np.floating)) or not 0.0 < th < 1.0:
            raise ValueError(f"threshold must be in (0, 1), got {th!r}")
        if isinstance(rs, bool) or not isinstance(rs, (int, float, np.integer, np.floating)) or \
                not math.isfinite(rs):
            raise ValueError(f"radius_scale must be a finite number, got {rs!r}")
        self.resolution, self.threshold, self.radius_scale = int(res), float(th), float(rs)
        self.ws_dir = _workspace(cfg)

    def __call__(self, model, dataset, overwrite=False):
        if overwrite or not os.path.exists(os.path.join(self.ws_dir, "visual_hull.ply")):
            self.construct_visual_hull(dataset, _device_of(model))
        return self.build_model(model)

    def construct_visual_hull(self, dataset, device="cuda"):
        cameras = list(dataset)
        if not cameras:
            raise ValueError("the dataset has no cameras")
        translate, extent = scene_extent(dataset, cameras)
        radius = extent * self.radius_scale
        occ = visual_hull_carve(cameras, self.resolution, radius, translate, device)
        if not bool(occ.any()):
            raise ValueError("the visual hull is empty: no grid node is inside every camera's mask")
        v, f = visual_hull_mesh(occ, self.threshold, radius, translate)
        if v.shape[0] == 0:
            raise ValueError("the visual hull has no surface: every grid node is inside every camera's mask")
        from .io import export_mesh_ply
        export_mesh_ply(os.path.join(self.ws_dir, "visual_hull.ply"), v, f)
        return v, f

    def build_model(self, model):
        from .io import load_mesh_ply
        dev = _device_of(model)
        xyz = load_mesh_ply(os.path.join(self.ws_dir, "visual_hull.ply"))[0].to(dev)
        P = xyz.shape[0]
        ones = lambda w: torch.ones((P, w), dtype=torch.float32, device=dev)
        model.create_from_attribute(xyz=xyz, rgb=ones(3) * 0.5, opacity=ones(1) * 0.1, scale=ones(3) * 0.01)
        return model


@register("depth")
class DepthInitializer(BaseInitializer):
    """depth.py:18-91: every view with a depth map, downsampled by 4, back-projected to world points (one row per
    pixel, depth 0 included), coloured by its image, scale depth / ((fx + fy) / 2); the reference's float16 round trip
    through `fused.ply` (double x y z of the float16 points, uchar colours trunc(float16(rgb16 * 255))) and
    `scales.bin` (raw float16) is kept exactly.  The model gets rgb = colour / 255, log-scale numpy's float16
    log(scale16) on all three axes (-inf where the depth is 0, as in the reference) and opacity logit 0.  When fused.ply exists and
    overwrite is False the model is built from the workspace; without scales.bin the scales come from dist2."""

    def __init__(self, config):
        super().__init__(config)
        self.ws_dir = _workspace(self.initializer_config)

    def __call__(self, model, dataset, overwrite=False):
        if overwrite or not os.path.exists(os.path.join(self.ws_dir, "fused.ply")):
            self.process_dataset(dataset, _device_of(model))
        return self.build_model(model)

    @staticmethod
    def prepare_views(dataset):
        """Copies of the cameras with a depth map, downsampled by 4 on the host; the caller's cameras are untouched."""
        views = []
        for cam in dataset:
            if cam.depth is None:
                continue
            if cam.image is None or cam.image.dim() != 3 or tuple(cam.image.shape[:2]) != tuple(cam.depth.shape):
                raise ValueError("a view with a depth map needs an image [H,W,3] of the same size, got "
                                 f"{None if cam.image is None else list(cam.image.shape)} for depth "
                                 f"{list(cam.depth.shape)}")
            views.append(copy.copy(cam).downsample_scale(4))
        if not views:
            raise ValueError("no camera has a depth map")
        return views

    def process_dataset(self, dataset, device="cuda"):
        """-> (xyz16 [N,3], colors uint8 [N,3], scale16 [N,1]) on device, also written to the workspace."""
        from .io import export_points_ply
        views = self.prepare_views(dataset)
        dev = torch.device(device)
        if dev.type != "cuda":
            raise ValueError("the depth initializer back-projects on the device: use a CUDA model")
        xyz, rgb, scale = [], [], []
        for cam in views:
            depth = cam.depth.to(dev, torch.float32).contiguous()
            xyz.append(cam.depth2point(depth, coordinate="world").reshape(-1, 3))
            rgb.append(cam.image.to(dev, torch.float32).reshape(-1, 3))
            scale.append((depth / ((cam.fx + cam.fy) / 2)).reshape(-1, 1))
        xyz16, rgb16, scale16 = (torch.cat(a).half() for a in (xyz, rgb, scale))
        colors = (rgb16 * 255).to(torch.uint8)
        export_points_ply(os.path.join(self.ws_dir, "fused.ply"), xyz16.double(), colors)
        scale16.cpu().numpy().tofile(os.path.join(self.ws_dir, "scales.bin"))
        return xyz16, colors, scale16

    def build_model(self, model):
        from .io import read_ply_vertices
        dev = _device_of(model)
        v = read_ply_vertices(os.path.join(self.ws_dir, "fused.ply"))
        xyz = torch.from_numpy(np.stack([v[k] for k in "xyz"], 1).astype(np.float32)).to(dev)
        colors = torch.from_numpy(np.stack([v[k] for k in ("red", "green", "blue")], 1).astype(np.uint8)).to(dev)
        rgb = colors.float() / 255.0
        log_scales = None
        path = os.path.join(self.ws_dir, "scales.bin")
        if os.path.exists(path):
            # numpy's float16 log, as the reference takes it: it is not float32 log rounded to float16 (numpy 2.3 on
            # x86-64 differs from that in 13265 of the 31743 positive finite float16 values), so it stays on the host
            log16 = np.log(np.fromfile(path, dtype=np.float16).reshape(-1, 1))
            log_scales = torch.from_numpy(log16).to(dev).repeat(1, 3).float()
        opacity = torch.zeros((xyz.shape[0], 1), dtype=torch.float32, device=dev)  # inverse_sigmoid(0.5)
        model.create_from_attribute(xyz=xyz, rgb=rgb, opacity=opacity, scale=log_scales)
        return model
