"""Gaussian initialization on the GPU: the initializers of gaustudio/pipelines/initializers/ that need no dataset
loader, behind the reference's registry surface (`initializers/__init__.py:10-24`).

  dist2(xyz)                         distCUDA2 of simple_knn: mean squared distance to the 3 nearest other points
  normal2rotation(normals)           pcd.py:12-37 (the raw quaternion of [R0 | R1 | n])
  make({"name": "pcd", "model_path": ...})           pcd.py:39-77
  make({"name": "mesh", "n_gaussians_per_surface_triangle": n})   mesh.py:74-250 (SuGaR placement)
  make({"name": "voxel", "voxel_size": s})           mesh.py:252-442

An initializer is called as the reference calls it, `init(model, mesh=None, dataset=None, overwrite=False)`; it fills
`model` (a GaussianPointCloud) through `create_from_attribute` and returns it.  The kernels are in csrc/gsr_init.cu
and csrc/gsr_clean.cu (MODE_DIST2); DESIGN.md 7j states the contract and the departures from the reference.
"""
from collections.abc import Mapping
import ctypes as C
import math
import os

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
