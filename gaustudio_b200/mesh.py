"""Mesh extraction on the GPU -- the part of gaustudio/scripts/extract_mesh.py after the render (lines 86-186), which the
reference runs on the host through vdbfusion (TSDF fusion + marching cubes) and open3d (`--clean`):

  TSDFVolume(voxel_size, sdf_trunc, space_carving=False)   vdbfusion.VDBVolume          extract_mesh.py:86
    .integrate(points, origin, valid=None)                  VDBVolume.integrate          extract_mesh.py:115
    .extract_triangle_mesh(min_weight=0.0)                  VDBVolume.extract_triangle_mesh   extract_mesh.py:145
  clean_mesh(vertices, faces, ratio=0.5)                    cluster_connected_triangles + filtering   :152-186
  extract_mesh(renderer, pcd, cameras, ...)                 the loop, extract_mesh.py:95-146

CUDA tensors in and out; a CPU tensor is an error.  The volume is sparse (8^3-voxel bricks in a device hash table) and
lives in one buffer of `capacity_bricks` bricks; running out is reported by `extract_triangle_mesh` with the capacity
the scene needs.  Integration never synchronises with the host; extraction reads its counts back once.

Rendering and colouring a mesh at a set of cameras -- what gaustudio/scripts/render_mesh.py and texture_mesh.py do
through pytorch3d's MeshRasterizer (faces_per_pixel=1, blur_radius=0) -- with a z-buffer triangle rasterizer on the
device (csrc/gsr_meshraster.cu; the contract is in include/gsr.h and DESIGN.md):

  rasterize(vertices, faces, camera, znear=None)         fragments.pix_to_face / zbuf           render_mesh.py:320
  vertex_normals(vertices, faces)                        Meshes.verts_normals_packed            render_mesh.py:65
  render_mesh(vertices, faces, camera, vertex_colors)    the loop body, render_mesh.py:284-359
  texture_mesh(vertices, faces, cameras, images)         texture_mesh.py:76-146

Camera values are read on the host (`extract._extrinsics_host` / `_intrinsics_host`); no call synchronises per view.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import ALLOC, call, ptr
from .extract import _extrinsics_host, _intrinsics_host, _need_cuda

_SCRATCH = 1  # slot of _lib.scratch


class TSDFVolume:
    """Truncated signed distance volume with vdbfusion's VDBVolume interface.  Voxel i covers [i, i+1) * voxel_size;
    samples are averaged with weight 1 each.  `space_carving` and weighting functions are not supported."""

    def __init__(self, voxel_size, sdf_trunc, space_carving=False, capacity_bricks=65536, device="cuda"):
        if space_carving:
            raise ValueError("TSDFVolume: space_carving is not supported")
        self.voxel_size, self.sdf_trunc = float(voxel_size), float(sdf_trunc)
        self.capacity_bricks = int(capacity_bricks)
        self.device = torch.device(device)
        nbytes = _lib.lib().gsr_tsdf_bytes(self.capacity_bricks)
        if nbytes == 0:
            raise ValueError(f"TSDFVolume: capacity_bricks must be in 1..262144, got {capacity_bricks}")
        self.state = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        call("gsr_tsdf_init", self.device, ptr(self.state), self.capacity_bricks, self.voxel_size, self.sdf_trunc)

    def integrate(self, points, origin, valid=None):
        """Fuse one view: `points` [..., 3] float32 CUDA, `origin` the sensor position (3 numbers on the host),
        `valid` an optional bool CUDA mask of points[..., 0]'s shape (False: skipped).  No host synchronisation."""
        _need_cuda(points, "points")
        pts = points.detach().reshape(-1, 3).float().contiguous()
        o = np.asarray(origin.detach().cpu() if isinstance(origin, torch.Tensor) else origin, np.float64).reshape(3)
        m = None
        if valid is not None:
            _need_cuda(valid, "valid")
            m = valid.detach().reshape(-1).to(torch.bool).contiguous()
            if m.numel() != pts.shape[0]:
                raise RuntimeError("TSDFVolume.integrate: valid must have one entry per point")
        call("gsr_tsdf_integrate", self.device, ptr(self.state), self.capacity_bricks, pts.shape[0], ptr(pts), ptr(m),
             float(o[0]), float(o[1]), float(o[2]))

    def extract_triangle_mesh(self, min_weight=0.0):
        """-> (vertices [V,3] float32, faces [F,3] int64), CUDA.  Cubes of voxel centres whose 8 corners all have
        weight > min_weight; faces point towards positive tsdf (the observed side)."""
        return _lib.call_mesh("gsr_tsdf_extract", self.device, ptr(self.state), self.capacity_bricks, float(min_weight))

    def export(self):
        """-> (brick_keys [n] int64, sums [n,512] int64, weights [n,512] int32) in key order: the raw volume state
        (key = ((bz + 2^20) << 42) | ((by + 2^20) << 21) | (bx + 2^20); voxel (x, y, z) at (z*8 + y)*8 + x; the mean
        sample is sums / weights * sdf_trunc / 2^20)."""
        with _lib.scratch(self.device):
            n = call("gsr_tsdf_export", self.device, ptr(self.state), self.capacity_bricks, ALLOC, _SCRATCH, None, None,
                     None)
            keys = torch.empty(n, dtype=torch.int64, device=self.device)
            sums = torch.empty(n, 512, dtype=torch.int64, device=self.device)
            weights = torch.empty(n, 512, dtype=torch.int32, device=self.device)
            call("gsr_tsdf_export", self.device, ptr(self.state), self.capacity_bricks, ALLOC, _SCRATCH, ptr(keys),
                 ptr(sums), ptr(weights))
        return keys, sums, weights


def face_components(faces, n_vertices):
    """Component label of every face (triangles joined by shared edges): the smallest face index of its component."""
    _need_cuda(faces, "faces")
    f = faces.detach().to(torch.int64).contiguous()
    labels = torch.empty(f.shape[0], dtype=torch.int64, device=f.device)
    with _lib.scratch(f.device):
        call("gsr_mesh_face_components", f.device, f.shape[0], ptr(f), int(n_vertices), ALLOC, _SCRATCH, ptr(labels))
    return labels


def clean_mesh(vertices, faces, ratio=0.5):
    """The `--clean` step of extract_mesh.py:152-186: keep the components (triangles joined by shared EDGES) with more
    than ratio * (largest component's) triangles, then drop unreferenced vertices.  Relative order of the remaining
    vertices and faces is kept.  -> (vertices, faces)."""
    _need_cuda(vertices, "vertices")
    if faces.shape[0] == 0:
        return vertices, faces
    labels = face_components(faces, vertices.shape[0])
    counts = torch.bincount(labels, minlength=faces.shape[0])
    keep_f = counts[labels].double() > ratio * counts.max().double()
    f = faces[keep_f]
    used = torch.zeros(vertices.shape[0], dtype=torch.bool, device=vertices.device)
    used[f.reshape(-1)] = True
    new_index = torch.cumsum(used.long(), 0) - 1
    return vertices[used], new_index[f]


def extract_mesh(renderer, pcd, cameras, voxel_size=0.01, sdf_trunc=0.04, min_weight=5, clean=False,
                 capacity_bricks=65536):
    """The loop of extract_mesh.py:95-146 (+ `--clean`): render every camera (no grad), take the median depth where
    the final opacity is >= 0.5, lift it to world points and fuse it, then run marching cubes.  The reference's
    striding (`cameras[::3]`) and downscaling are the caller's choice, as in `extract.extract_pcd`.
    -> (vertices [V,3] float32, faces [F,3] int64), CUDA."""
    device = pcd._anchor.device if hasattr(pcd, "_anchor") else pcd._xyz.device  # Scaffold-GS anchors, or Gaussians
    volume = TSDFVolume(voxel_size, sdf_trunc, capacity_bricks=capacity_bricks, device=device)
    for camera in cameras:
        with torch.no_grad():
            pkg = renderer.render(camera, pcd)
        integrate_view(volume, camera, pkg["rendered_median_depth"][0], pkg["rendered_final_opacity"][0])
    vertices, faces = volume.extract_triangle_mesh(min_weight=min_weight)
    if clean:
        vertices, faces = clean_mesh(vertices, faces)
    return vertices, faces


def integrate_view(volume, camera, median_depth, opacity):
    """One view of the loop: world points of the whole median-depth map, `opacity >= 0.5` as the mask, the camera
    centre (inverse(extrinsics)[:3, 3], from the host copy of the extrinsics) as the origin.  No host synchronisation:
    no boolean compaction, and the camera-to-world matrix goes up through pinned memory."""
    from . import ops
    _need_cuda(median_depth, "median_depth")
    c2w = np.linalg.inv(_extrinsics_host(camera).astype(np.float64))
    fx, fy, cx, cy = _intrinsics_host(camera)
    m = torch.from_numpy(c2w.astype(np.float32)).pin_memory().to(median_depth.device, non_blocking=True)
    pts = ops.depth2point(median_depth.detach(), fx, fy, cx, cy, m)
    volume.integrate(pts, c2w[:3, 3], valid=opacity >= 0.5)


# ---- mesh rendering and texturing ----
_RASTER_SCRATCH = {}


def _camera_host(camera):
    """-> (12 doubles R|t of the world->camera transform, (fx, fy, cx, cy), W, H), all from host copies."""
    E = _extrinsics_host(camera).astype(np.float64)
    rt = np.ascontiguousarray(np.concatenate([E[:3, :3].ravel(), E[:3, 3]]), np.float64)
    return rt, tuple(float(x) for x in _intrinsics_host(camera)), int(camera.image_width), int(camera.image_height)


def _raster_scratch(device, W, H, nbytes):
    """The rasterizer's scratch for (device, stream, W, H), grown when a mesh needs more.  A new one starts with every
    byte 0xff (the empty z-buffer); each rasterize leaves its z-buffer empty again, so it is never cleared after that."""
    key = (device, _lib.stream(device), W, H)
    s = _RASTER_SCRATCH.get(key)
    if s is None or s.numel() < nbytes:
        s = torch.full((nbytes,), 255, dtype=torch.uint8, device=device)
        _RASTER_SCRATCH[key] = s
    return s


def _mesh_tensors(vertices, faces):
    _need_cuda(vertices, "vertices")
    _need_cuda(faces, "faces")
    v = vertices.detach().reshape(-1, 3).float().contiguous()
    f = faces.detach().reshape(-1, 3).to(device=v.device, dtype=torch.int64).contiguous()
    return v, f


def rasterize(vertices, faces, camera, znear=None):
    """Hard z-buffer of a triangle mesh at `camera` (pytorch3d MeshRasterizer, faces_per_pixel=1, blur_radius=0, no
    culling): vertices [V,3] float32, faces [F,3] int64 CUDA.  Pixel (column i, row j) samples the image point (i, j),
    the frame of Camera.depth2point.  Faces with an index outside [0, V), a vertex at z <= znear (default:
    camera.znear) or outside the 2^20-px guard band, or zero area are not drawn.
    -> (face_id [H,W] int32, -1 where no face; depth [H,W] float32 view z, -1 where no face)."""
    v, f = _mesh_tensors(vertices, faces)
    rt, (fx, fy, cx, cy), W, H = _camera_host(camera)
    zn = float(camera.znear if znear is None else znear)
    nbytes = _lib.lib().gsr_mesh_raster_bytes(v.shape[0], f.shape[0], W, H)
    if nbytes == 0:
        raise ValueError(f"rasterize: unsupported sizes (V={v.shape[0]}, F={f.shape[0]}, {W}x{H})")
    scratch = _raster_scratch(v.device, W, H, nbytes)
    face_id = torch.empty(H, W, dtype=torch.int32, device=v.device)
    depth = torch.empty(H, W, dtype=torch.float32, device=v.device)
    call("gsr_mesh_rasterize", v.device, v.shape[0], ptr(v), f.shape[0], ptr(f), rt.ctypes.data_as(C.c_void_p), fx,
         fy, cx, cy, zn, W, H, ptr(scratch), scratch.numel(), ptr(face_id), ptr(depth))
    return face_id, depth


def vertex_normals(vertices, faces):
    """pytorch3d's verts_normals_packed: every vertex sums the cross products of its corners' two edges, normalised
    with eps 1e-6.  [V,3] float32 CUDA; built once per mesh."""
    v, f = _mesh_tensors(vertices, faces)
    vf = v[f]
    n = torch.zeros_like(v)
    for i in range(3):
        j, k = (i + 1) % 3, (i + 2) % 3
        n.index_add_(0, f[:, i], torch.linalg.cross(vf[:, j] - vf[:, i], vf[:, k] - vf[:, i], dim=1))
    return torch.nn.functional.normalize(n, eps=1e-6, dim=1)


def render_mesh(vertices, faces, camera, vertex_colors=None, normals=None, znear=None):
    """One view of render_mesh.py:284-359 -> {face_id, depth, mask [H,W] bool, normal [H,W,3], color [H,W,3]}.
    normal: normalize(n_a + n_b + n_c) of the hit face's vertex normals (`normals`, default vertex_normals(...); pass
    them in when rendering many views) rotated into the camera frame, 0 where no face -- the reference interpolates
    with barycentrics of ones.  color: perspective-correct interpolation of vertex_colors [V,3], 1 on a hit without
    colours, 0 where no face.  The y/z sign flip and PNG encoding of the script are the caller's."""
    v, f = _mesh_tensors(vertices, faces)
    face_id, depth = rasterize(v, f, camera, znear)
    rt, (fx, fy, cx, cy), W, H = _camera_host(camera)
    n = (vertex_normals(v, f) if normals is None else normals).detach().float().contiguous()
    col = None if vertex_colors is None else vertex_colors.detach().to(v.device).float().contiguous()
    for t, what in ((n, "normals"), (col, "vertex_colors")):
        if t is not None and tuple(t.shape) != (v.shape[0], 3):
            raise ValueError(f"render_mesh: {what} must be [V,3]")
    normal = torch.empty(H, W, 3, dtype=torch.float32, device=v.device)
    color = torch.empty(H, W, 3, dtype=torch.float32, device=v.device)
    call("gsr_mesh_shade", v.device, v.shape[0], ptr(v), f.shape[0], ptr(f), rt.ctypes.data_as(C.c_void_p), fx, fy,
         cx, cy, W, H, ptr(face_id), ptr(n), ptr(col), ptr(normal), ptr(color))
    return {"face_id": face_id, "depth": depth, "mask": face_id >= 0, "normal": normal, "color": color}


def texture_mesh(vertices, faces, cameras, images, znear=None):
    """Vertex colours from the views' images (texture_mesh.py:76-146): per view, the faces that own a pixel and face
    the camera (cos(normal, optical axis) < -0.05) stamp their vertices; each stamped vertex inside the image gets
    clamp(bilinear(image, u, v), 0, 1), the last view winning; vertices never written stay 0.  images: float [H,W,3]
    per camera.  Raises after the loop, naming the first view whose visible faces have a non-negative mean cosine (the
    reference's assertion; a view with no visible face is skipped).  -> vertex_colors [V,3] float32 CUDA."""
    v, f = _mesh_tensors(vertices, faces)
    V, F = v.shape[0], f.shape[0]
    face_stamp = torch.zeros(F, dtype=torch.int32, device=v.device)
    vertex_stamp = torch.zeros(V, dtype=torch.int32, device=v.device)
    colors = torch.zeros(V, 3, dtype=torch.float32, device=v.device)
    cameras = list(cameras)
    stats = torch.zeros(len(cameras), 2, dtype=torch.int64, device=v.device)
    for i, (camera, image) in enumerate(zip(cameras, images)):
        face_id, _ = rasterize(v, f, camera, znear)
        rt, (fx, fy, cx, cy), W, H = _camera_host(camera)
        _need_cuda(image, "images")
        img = image.detach().to(v.device).float().contiguous()
        if tuple(img.shape) != (H, W, 3):
            raise ValueError(f"texture_mesh: image {i} is {tuple(img.shape)}, expected ({H}, {W}, 3)")
        call("gsr_mesh_texture_view", v.device, V, ptr(v), F, ptr(f), rt.ctypes.data_as(C.c_void_p), fx, fy, cx, cy,
             W, H, ptr(face_id), ptr(img), i, ptr(face_stamp), ptr(vertex_stamp), ptr(stats[i]), ptr(colors))
    for i, (q, n) in enumerate(stats.cpu().tolist()):
        if n > 0 and q >= 0:
            raise RuntimeError(f"texture_mesh: view {i}: the visible faces' normals point away from the camera on "
                               f"average (mean cos {q / 2.0**40 / n:.4f} >= 0); are the faces flipped?")
    return colors
