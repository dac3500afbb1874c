"""Extraction post-pass on the GPU -- the step right after the rasterizer in gaustudio/scripts/extract_pcd.py
(SURVEY.md 8f row 2).  Same function names, argument meaning and results as the reference script:

  masked_bilateral_filter(depth_map, mask, d, sigma_color, sigma_space)      extract_pcd.py:185-238
  normal_fusion(pcd, all_ids_list, all_normals_list, all_confidences_list, cameras)   extract_pcd.py:108-183
  getNerfppNorm(cameras)                                                     gaustudio/datasets/utils.py:82-104
  extract_view(camera, render_pkg, scene_radius)                             the loop body, extract_pcd.py:314-337
  extract_pcd(renderer, pcd, cameras)                                        the loop + fusion, extract_pcd.py:309-345
  mesh_sap(xyz, normals, res=256, sig=2)                                     `--meshing sap`, extract_pcd.py:102-106
  dpsr(points01, normals, res, sig)                                          models/sap.py + utils/graphics_utils.py DPSR
  clean_point_cloud(xyz, rgb, normals)                                       extract_pcd.py:46-51
  remove_statistical_outlier(xyz, nb_neighbors, std_ratio)                   Open3D's, called at extract_pcd.py:47
  remove_normal_outliers(xyz, normals, nb_neighbors, angle_threshold)        extract_pcd.py:30-43

The reference moves every depth map to the host for OpenCV (dilate + bilateralFilter) and back; here the filter,
the normal extraction and the fusion passes are CUDA kernels behind the C ABI (include/gsr.h) and nothing is
synchronised per view.  The k-nearest-neighbour search of the final smoothing (scipy's cKDTree on the host in the
reference) is a uniform-grid search on the device as well (`knn`, gsr_knn_grid).  The Shape-as-Points meshing (DPSR
Poisson solve + marching cubes) is CUDA kernels around torch's cuFFT (csrc/gsr_sap.cu, DESIGN.md 7h), and the
point-cloud cleaning an exact k-nearest-neighbour search fused with its two consumers (csrc/gsr_clean.cu, DESIGN.md 7i).
"""
import math

import numpy as np
import torch

from . import _lib
from ._lib import ALLOC, call, ptr


def _need_cuda(t, what):
    if not (isinstance(t, torch.Tensor) and t.is_cuda):
        raise RuntimeError(f"{what} must be a CUDA tensor (the extraction post-pass has no CPU path)")


def _extrinsics_host(camera):
    """float32 numpy copy of camera.extrinsics without touching the device when the camera keeps R / T on the host
    (world_view_transform = [[R^T, T], [0, 1]] up to the recentring of datasets/__init__.py:52-64, which only moves
    the translation)."""
    wvt = getattr(camera, "world_view_transform", None)
    if isinstance(wvt, torch.Tensor) and not wvt.is_cuda:
        return wvt.transpose(0, 1).contiguous().numpy().astype(np.float32)
    if getattr(camera, "trans", None) is not None and np.allclose(camera.trans, 0) and getattr(camera, "scale", 1.0) == 1.0:
        E = np.eye(4, dtype=np.float32)
        E[:3, :3] = np.asarray(camera.R, np.float32).T
        E[:3, 3] = np.asarray(camera.T, np.float32)
        return E
    return camera.extrinsics.detach().cpu().numpy().astype(np.float32)


def masked_bilateral_filter(depth_map, mask, d=3, sigma_color=75, sigma_space=75):
    """Bilateral-filter the valid part of a depth map; returns (filtered_depth, new_mask) where new_mask marks
    pixels whose d x d window is entirely valid.  [H,W] float32 / bool CUDA tensors in and out."""
    _need_cuda(depth_map, "depth_map")
    if depth_map.dim() != 2:
        raise RuntimeError("masked_bilateral_filter expects an [H,W] depth map")
    depth = depth_map.detach().float().contiguous()
    m = mask.detach().to(device=depth.device, dtype=torch.bool).contiguous()
    H, W = depth.shape
    out = torch.empty_like(depth)
    new_mask = torch.empty(H, W, dtype=torch.bool, device=depth.device)
    scratch = torch.empty(2, dtype=torch.int32, device=depth.device)
    call("gsr_masked_bilateral", depth.device, ptr(depth), ptr(m), W, H, int(d), float(sigma_color),
         float(sigma_space), ptr(out), ptr(new_mask), ptr(scratch))
    return out, new_mask.to(mask.dtype)


def getNerfppNorm(cameras):
    """Scene centre / radius from the camera centres (gaustudio/datasets/utils.py:82-104)."""
    centres = []
    for cam in cameras:
        w2c = np.eye(4)
        w2c[:3, :3] = np.asarray(cam.R, np.float64).T
        w2c[:3, 3] = np.asarray(cam.T, np.float64)
        centres.append(np.linalg.inv(w2c)[:3, 3:4])
    centres = np.hstack(centres)
    centre = centres.mean(axis=1, keepdims=True)
    dist = np.linalg.norm(centres - centre, axis=0)
    return {"translate": -centre.flatten(), "radius": float(dist.max() * 1.1), "min_radius": float(dist.min() * 1.5)}


def _intrinsics_host(camera):
    """(fx, fy, cx, cy) as host floats without touching the device: from the camera's FoV / size / principal point
    (the formula of Camera.intrinsics, gaustudio/datasets/__init__.py:229-237) when it has them."""
    if all(hasattr(camera, a) for a in ("FoVx", "FoVy", "image_width", "image_height")):
        W, H = int(camera.image_width), int(camera.image_height)
        pp = getattr(camera, "principal_point_ndc", None)
        px, py = (0.5, 0.5) if pp is None else (float(pp[0]), float(pp[1]))
        return (W / (2.0 * math.tan(camera.FoVx / 2.0)), H / (2.0 * math.tan(camera.FoVy / 2.0)), W * px, H * py)
    K = camera.intrinsics  # a device-resident K costs one synchronising read here
    return float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])


def extract_view(camera, render_pkg, scene_radius, d=3, sigma_color=75, sigma_space=75, compact=True):
    """One view of the extraction loop.  Returns dict(filtered_depth, fg_mask, cam_normals [H,W,3], valid [H,W],
    ids [n] int64, normals [n,3] (negated world normals), confidences [n]).

    compact=True gathers the valid pixels like the reference (`ids[valid]`: a boolean-mask gather, i.e. one stream
    synchronisation per view).  compact=False is sync-free: ids / normals / confidences cover ALL H*W pixels and the
    invalid ones carry id -1, which `normal_fusion` skips (negative ids mean "no observation" there)."""
    opacity = render_pkg["rendered_final_opacity"][0].contiguous()
    depth = render_pkg["rendered_depth"][0]
    median_depth = render_pkg["rendered_median_depth"][0].contiguous()
    median_ids = render_pkg["rendered_median_id"][0]
    _need_cuda(opacity, "render_pkg tensors")
    dev = opacity.device
    H, W = opacity.shape
    filtered, fg = masked_bilateral_filter(depth, opacity > 0.1, d, sigma_color, sigma_space)
    fx, fy, cx, cy = _intrinsics_host(camera)
    rot = torch.from_numpy(np.ascontiguousarray(np.linalg.inv(_extrinsics_host(camera)[:3, :3]).T)).to(dev)
    cam_normals = torch.empty(H, W, 3, dtype=torch.float32, device=dev)
    neg_world = torch.empty(H, W, 3, dtype=torch.float32, device=dev)
    valid = torch.empty(H, W, dtype=torch.bool, device=dev)
    call("gsr_extract_normals", dev, ptr(filtered), ptr(fg), ptr(opacity), ptr(median_depth), W, H, float(fx),
         float(fy), float(cx), float(cy), ptr(rot), float(scene_radius * 0.8), 0.5, ptr(cam_normals), ptr(neg_world),
         ptr(valid))
    res = {"filtered_depth": filtered, "fg_mask": fg, "cam_normals": cam_normals, "valid": valid}
    if compact:
        res.update(ids=median_ids[valid].long(), normals=neg_world[valid], confidences=opacity[valid])
    else:
        res.update(ids=torch.where(valid, median_ids.long(), -1).reshape(-1), normals=neg_world.reshape(-1, 3),
                   confidences=opacity.reshape(-1))
    return res


def _fusion_pass(xyz, ids_list, normals_list, conf_list, cam_ts, mean, sums, weights, touched):
    dev = xyz.device
    for ids, n, c, t in zip(ids_list, normals_list, conf_list, cam_ts):
        if ids.numel() == 0:
            continue
        ids = ids.to(device=dev, dtype=torch.int64).contiguous()
        n = n.to(device=dev, dtype=torch.float32).contiguous()
        c = c.to(device=dev, dtype=torch.float32).contiguous()
        call("gsr_normal_fusion_pass", dev, ids.numel(), ptr(ids), ptr(n), ptr(c), xyz.shape[0], ptr(xyz), t[0], t[1],
             t[2], ptr(mean), 0.8, ptr(sums), ptr(weights), ptr(touched))
    out = torch.empty_like(sums)
    call("gsr_normal_fusion_mean", dev, xyz.shape[0], ptr(sums), ptr(weights), ptr(out))
    return out


def normal_fusion(pcd, all_ids_list, all_normals_list, all_confidences_list, cameras, smooth=True):
    """Weighted, consistency-checked fusion of per-view normals into one normal per observed Gaussian.
    Returns (unique_ids ascending, normals [n,3]) like the reference.
    Ids outside [0, P) are skipped: negative ids are the "no observation" sentinel of `extract_view(compact=False)`.
    (The reference indexes `pcd._xyz[ids]` with them: -1 wraps to the last Gaussian and ids >= P raise; its own loop
    never produces either, extract_pcd.py:325-337.)"""
    xyz = pcd._xyz.detach().float().contiguous()
    _need_cuda(xyz, "pcd._xyz")
    dev, P = xyz.device, xyz.shape[0]
    # what the reference uses as the camera position: extrinsics[:3, 3] (taken from the host copy of R / T)
    cam_ts = [_extrinsics_host(cam)[:3, 3].tolist() for cam in cameras]
    sums = torch.zeros(P, 3, device=dev); weights = torch.zeros(P, device=dev)
    touched = torch.zeros(P, dtype=torch.uint8, device=dev)
    mean = _fusion_pass(xyz, all_ids_list, all_normals_list, all_confidences_list, cam_ts, None, sums, weights, touched)
    sums.zero_(); weights.zero_()
    mean = _fusion_pass(xyz, all_ids_list, all_normals_list, all_confidences_list, cam_ts, mean, sums, weights, None)
    unique_ids = torch.nonzero(touched, as_tuple=False).flatten()
    mean = mean[unique_ids]
    if not smooth or unique_ids.numel() == 0:
        return unique_ids, mean
    # spatial smoothing over the 10 nearest surface points (extract_pcd.py:170-181: scipy cKDTree on the host there);
    # here the neighbour search stays on the device (the reference needs >= 10 surface points)
    dist, idx = knn(xyz[unique_ids], k=min(10, int(unique_ids.numel())))
    w = torch.exp(-dist.double() / 0.1)
    sm = (mean[idx].double() * w.unsqueeze(-1)).sum(1).float()
    return unique_ids, torch.nn.functional.normalize(sm, p=2, dim=1)


_KNN_K = (1, 4, 8, 10, 16)


def knn(points, k=10):
    """k nearest neighbours of every point among `points` [n,3] (float32, CUDA) -> (dist [n,k] float32, idx [n,k] int64),
    ascending distance with the point itself first -- what `cKDTree(points).query(points, k)` returns
    (extract_pcd.py:170-171), without leaving the device.  Uniform-grid search (gsr_knn_grid): the points are sorted by
    cell with torch ops, the bounding box / cell size never come back to the host."""
    _need_cuda(points, "points")
    pts = points.detach().float().contiguous()
    n, dev = pts.shape[0], pts.device
    if k not in _KNN_K or n <= k:  # tiny inputs / unusual k: exact all-pairs search (still on the device)
        d = torch.cdist(pts.double(), pts.double())
        dist, idx = d.topk(min(k, n), dim=1, largest=False)
        return dist.float(), idx
    G = min(256, max(8, 1 << math.ceil(math.log2(max(n, 2) ** (1.0 / 3.0)))))
    lo, hi = pts.min(dim=0).values, pts.max(dim=0).values
    ext = (hi - lo).clamp_min(1e-12)
    inv_h = 1.0 / (ext.max() / G * 1.0001 + 1e-12)
    dims = torch.clamp(torch.ceil(ext * inv_h), min=1.0, max=float(G))
    cell = torch.minimum(torch.clamp(((pts - lo) * inv_h).floor(), min=0.0), dims - 1.0)
    cid = ((cell[:, 2] * dims[1] + cell[:, 1]) * dims[0] + cell[:, 0]).long()
    order = torch.argsort(cid, stable=True)
    sorted_pts = pts[order].contiguous()
    counts = torch.zeros(G ** 3 + 1, dtype=torch.int64, device=dev)
    counts.scatter_add_(0, cid + 1, torch.ones_like(cid))
    cell_start = torch.cumsum(counts, 0).to(torch.int32).contiguous()
    grid = torch.cat([lo, inv_h.reshape(1), dims, torch.zeros(1, device=dev)]).float().contiguous()
    out_i = torch.empty(n, k, dtype=torch.int32, device=dev)
    out_d = torch.empty(n, k, dtype=torch.float32, device=dev)
    call("gsr_knn_grid", dev, n, k, ptr(sorted_pts), ptr(cell_start), ptr(grid), ptr(out_i), ptr(out_d))
    dist = torch.empty_like(out_d)
    idx = torch.empty(n, k, dtype=torch.int64, device=dev)
    dist[order] = out_d                     # rows back to the caller's order ...
    idx[order] = order[out_i.long()]        # ... and neighbour indices back to the caller's numbering
    return dist, idx


def SH2RGB(sh):
    """gaustudio/utils/sh_utils.py:114-118."""
    return sh * 0.28209479177387814 + 0.5


def extract_pcd(renderer, pcd, cameras, d=3, sigma_color=75, sigma_space=75, smooth=True):
    """Render every camera and fuse a surface point cloud: (xyz [n,3], rgb [n,3], normals [n,3], per-view results).
    The loop of extract_pcd.py:309-345 without its image / .cam file output and without meshing."""
    scene_radius = getNerfppNorm(cameras)["radius"]
    ids_l, nrm_l, conf_l, views = [], [], [], []
    for camera in cameras:
        with torch.no_grad():
            pkg = renderer.render(camera, pcd)
        v = extract_view(camera, pkg, scene_radius, d, sigma_color, sigma_space, compact=False)  # no per-view sync
        ids_l.append(v["ids"]); nrm_l.append(v["normals"]); conf_l.append(v["confidences"])
        views.append(v)
    unique_ids, normals = normal_fusion(pcd, ids_l, nrm_l, conf_l, cameras, smooth=smooth)
    f_dc = pcd._f_dc[unique_ids]
    rgb = SH2RGB(f_dc.reshape(f_dc.shape[0], -1)[:, :3]).clip(0, 1)
    return pcd._xyz[unique_ids], rgb, normals, views


# ---- Shape-as-Points meshing: the `--meshing sap` step of extract_pcd.py:397-399 (models/sap.py, DPSR) ----
_SAP_SCRATCH = 1  # slot of _lib.scratch


def _sap_inputs(points, normals, res, sig, what):
    """Refuses bad input before any device work (the device is checked last, so every other refusal also fires on CPU
    tensors); -> (points, normals) contiguous."""
    for t, name in ((points, what), (normals, "normals")):
        if not isinstance(t, torch.Tensor):
            raise ValueError(f"{name} must be a tensor")
        if t.dtype != torch.float32:
            raise ValueError(f"{name} must be float32, got {t.dtype}")
        if t.dim() != 2 or t.shape[1] != 3:
            raise ValueError(f"{name} must be [N,3], got {tuple(t.shape)}")
    if points.shape != normals.shape or points.device != normals.device:
        raise ValueError(f"{what} and normals must have the same shape and device")
    if points.shape[0] == 0:
        raise ValueError(f"{what} must hold at least one point")
    if points.shape[0] > 2**31 - 1:
        raise ValueError(f"{what} holds more than 2^31-1 points")
    if isinstance(res, bool) or not isinstance(res, (int, np.integer)) or not 2 <= res <= 512:
        raise ValueError(f"res must be an integer in 2..512, got {res!r}")
    if not (isinstance(sig, (int, float, np.integer, np.floating)) and math.isfinite(sig) and sig > 0):
        raise ValueError(f"sig must be positive and finite, got {sig!r}")
    if not points.is_cuda:
        raise ValueError(f"{what} and normals must be CUDA tensors (Shape-as-Points meshing has no CPU path)")
    return points.detach().contiguous(), normals.detach().contiguous()


def _sap_splat(points01, normals, res):
    """point_rasterize(points01, normals, res, weighted=False) -> [3,res,res,res] float32 (no argument checks)."""
    grid = torch.empty(3, res, res, res, dtype=torch.float32, device=points01.device)
    with _lib.scratch(points01.device):
        call("gsr_sap_splat", points01.device, points01.shape[0], ptr(points01), ptr(normals), int(res), ALLOC,
             _SAP_SCRATCH, ptr(grid))
    return grid


def _sap_psi(points01, normals, res, sig):
    dev = points01.device
    grid = _sap_splat(points01, normals, res)
    spectrum = torch.fft.rfftn(grid, dim=(1, 2, 3))  # cuFFT
    del grid
    phi_hat = torch.empty(res, res, res // 2 + 1, dtype=torch.complex64, device=dev)
    call("gsr_sap_spectral", dev, int(res), float(sig), ptr(spectrum), ptr(phi_hat))
    del spectrum
    phi = torch.fft.irfftn(phi_hat, s=(res, res, res)).contiguous()
    del phi_hat
    psi = torch.empty_like(phi)
    with _lib.scratch(dev):
        call("gsr_sap_shift_scale", dev, points01.shape[0], ptr(points01), int(res), ptr(phi), ALLOC, _SAP_SCRATCH,
             ptr(psi))
    return psi


def dpsr(points01, normals, res=256, sig=2):
    """DPSR(res, sig, scale=True, shift=True, weighted=False) of gaustudio/utils/graphics_utils.py followed by the tanh
    of ShapeAsPoints.generate_mesh: the grid psi [res,res,res] float32, indexed [x,y,z] with node k at k/res, positive
    outside the shape (where the normals point) and negative inside, as the reference's.  points01 [N,3] in [0,1) and normals [N,3], float32 CUDA."""
    p, n = _sap_inputs(points01, normals, res, sig, "points01")
    ok = torch.stack([torch.isfinite(p).all() & torch.isfinite(n).all(), ((p >= 0) & (p < 1)).all()]).cpu()
    if not ok[0]:
        raise ValueError("points01 and normals must be finite")
    if not ok[1]:
        raise ValueError("points01 must lie in [0, 1)")
    return _sap_psi(p, n, int(res), float(sig))


def mesh_sap(xyz, normals, res=256, sig=2):
    """The `--meshing sap` step of extract_pcd.py (mesh_sap -> ShapeAsPoints.from_o3d_pointcloud + generate_mesh):
    normalise the oriented points into the unit cube, DPSR at `res` / `sig`, marching cubes of the tanh'd grid at 0,
    and the vertices mapped back to world coordinates.  xyz, normals: [N,3] float32 CUDA, finite (drop NaN-normal rows
    first), not all the same point.  -> (vertices [V,3] float32, faces [F,3] int64), CUDA; faces face outward."""
    x, n = _sap_inputs(xyz, normals, res, sig, "xyz")
    ok = torch.stack([torch.isfinite(x).all() & torch.isfinite(n).all(), (x != x[:1]).any()]).cpu()
    if not ok[0]:
        raise ValueError("xyz and normals must be finite")
    if not ok[1]:
        raise ValueError("xyz must hold at least two distinct points (their spread sets the grid's scale)")
    dev, res = x.device, int(res)
    points01 = torch.empty_like(x)
    transform = torch.empty(4, dtype=torch.float32, device=dev)
    with _lib.scratch(dev):
        call("gsr_sap_normalize", dev, x.shape[0], ptr(x), ALLOC, _SAP_SCRATCH, ptr(points01), ptr(transform))
    psi = _sap_psi(points01, n, res, float(sig))
    return _lib.call_mesh("gsr_sap_marching_cubes", dev, res, ptr(psi), ptr(transform))


# ---- point-cloud cleaning: clean_point_cloud of extract_pcd.py:30-51 (csrc/gsr_clean.cu, DESIGN.md 7i) ----
_CLEAN_SCRATCH = 1  # slot of _lib.scratch


def _clean_inputs(xyz, normals, nb_neighbors):
    """Refuses bad input before any device work (the caller checks the device last, as _sap_inputs does).  The
    finiteness of xyz is read back from the device together with the survivor count."""
    for t, name in ((xyz, "xyz"), (normals, "normals")):
        if t is None:
            continue
        if not isinstance(t, torch.Tensor):
            raise ValueError(f"{name} must be a tensor")
        if t.dtype != torch.float32:
            raise ValueError(f"{name} must be float32, got {t.dtype}")
        if t.dim() != 2 or t.shape[1] != 3:
            raise ValueError(f"{name} must be [N,3], got {tuple(t.shape)}")
    if normals is not None and (normals.shape != xyz.shape or normals.device != xyz.device):
        raise ValueError("xyz and normals must have the same shape and device")
    if xyz.shape[0] > 2**31 - 1:
        raise ValueError("xyz holds more than 2^31-1 points")
    if isinstance(nb_neighbors, bool) or not isinstance(nb_neighbors, (int, np.integer)) or not 1 <= nb_neighbors <= 64:
        raise ValueError(f"nb_neighbors must be an integer in 1..64, got {nb_neighbors!r}")


def _on_cuda(xyz, what):
    if not xyz.is_cuda:
        raise ValueError(f"{what} must be CUDA tensors (point-cloud cleaning has no CPU path)")


def _survivors(keep, xyz):
    """Ascending int64 indices of keep != 0: one read of (count, xyz finite) sizes the compaction.  Non-finite xyz is
    therefore refused after the pass has run on it (the kernels stay in bounds and terminate on NaN / inf), not before
    any device work as the other refusals are."""
    cnt, finite = torch.stack([keep.sum(dtype=torch.int64), torch.isfinite(xyz).all().long()]).tolist()
    if not finite:
        raise ValueError("xyz must be finite")
    return torch.nonzero_static(keep, size=cnt).flatten()


def remove_statistical_outlier(xyz, nb_neighbors=50, std_ratio=2.0):
    """Open3D's PointCloud.remove_statistical_outlier(nb_neighbors, std_ratio) on xyz [N,3] float32 CUDA: the ascending
    int64 indices of the points whose mean distance to their nb_neighbors nearest points (themselves included) is
    > 0 and < mean + std_ratio * std over the cloud (std with Bessel's correction over N).  Raises ValueError for
    non-finite xyz after the pass has run (the check shares the pass's one read-back)."""
    _clean_inputs(xyz, None, nb_neighbors)
    if not (isinstance(std_ratio, (int, float, np.integer, np.floating)) and not isinstance(std_ratio, bool)
            and math.isfinite(std_ratio) and std_ratio > 0):
        raise ValueError(f"std_ratio must be positive and finite, got {std_ratio!r}")
    _on_cuda(xyz, "xyz")
    x, dev, n = xyz.detach().contiguous(), xyz.device, xyz.shape[0]
    if n == 0:
        return torch.empty(0, dtype=torch.int64, device=dev)
    avg = torch.empty(n, dtype=torch.float64, device=dev)
    stats = torch.empty(3, dtype=torch.float64, device=dev)
    keep = torch.empty(n, dtype=torch.uint8, device=dev)
    with _lib.scratch(dev):
        call("gsr_clean_statistical", dev, n, ptr(x), int(nb_neighbors), float(std_ratio), ALLOC, _CLEAN_SCRATCH,
             ptr(avg), ptr(stats), ptr(keep))
    return _survivors(keep, x)


def remove_normal_outliers(xyz, normals, nb_neighbors=20, angle_threshold=math.pi / 4):
    """remove_normal_outliers of extract_pcd.py:30-43 on xyz / normals [N,3] float32 CUDA: the ascending int64 indices of
    the points whose mean acos(|n_i . n_j|) over their nb_neighbors - 1 nearest other points is < angle_threshold.
    |dot| is clamped to 1 (the reference's arccos turns the float32 |n|^2 > 1 of parallel normals into NaN); NaN
    normals are accepted and drop the points whose neighbourhood holds one.  Non-finite xyz raises ValueError after
    the pass has run."""
    _clean_inputs(xyz, normals, nb_neighbors)
    if not (isinstance(angle_threshold, (int, float, np.integer, np.floating)) and not isinstance(angle_threshold, bool)
            and math.isfinite(angle_threshold)):
        raise ValueError(f"angle_threshold must be finite, got {angle_threshold!r}")
    _on_cuda(xyz, "xyz and normals")
    x, nr, dev, n = xyz.detach().contiguous(), normals.detach().contiguous(), xyz.device, xyz.shape[0]
    if n == 0:
        return torch.empty(0, dtype=torch.int64, device=dev)
    mean_angle = torch.empty(n, dtype=torch.float64, device=dev)
    keep = torch.empty(n, dtype=torch.uint8, device=dev)
    with _lib.scratch(dev):
        call("gsr_clean_normal", dev, n, ptr(x), ptr(nr), int(nb_neighbors), float(angle_threshold), ALLOC,
             _CLEAN_SCRATCH, ptr(mean_angle), ptr(keep))
    return _survivors(keep, x)


def clean_point_cloud(xyz, rgb, normals, nb_neighbors=50, std_ratio=2.0):
    """clean_point_cloud of extract_pcd.py:46-51: remove_statistical_outlier(nb_neighbors, std_ratio), then
    remove_normal_outliers(20, pi/4) on its survivors.  xyz / normals [N,3] float32 CUDA, rgb [N,...] on the same
    device.  -> (xyz, rgb, normals, index) with index the ascending int64 indices of the kept points."""
    if not isinstance(rgb, torch.Tensor) or not isinstance(xyz, torch.Tensor) or rgb.shape[:1] != xyz.shape[:1]:
        raise ValueError("rgb must be a tensor with one row per point")
    _clean_inputs(xyz, normals, nb_neighbors)
    if rgb.device != xyz.device:
        raise ValueError("rgb must be on the device of xyz")
    first = remove_statistical_outlier(xyz, nb_neighbors, std_ratio)
    second = remove_normal_outliers(xyz[first].contiguous(), normals[first].contiguous(), 20, math.pi / 4)
    index = first[second]
    return xyz[index], rgb[index], normals[index], index
