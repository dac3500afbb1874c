"""CPU restatement (numpy) of the reference's mesh / point-cloud extraction post-pass -- SURVEY.md section 8f row 2.

TEST INFRASTRUCTURE ONLY: imported by tests/ (and nothing in the product path).  Pinned against outputs of the
reference's own functions executed in the build container (tests/golden/extract_golden.npz, generator
tests/golden/make_golden_extract.py).  Follows

  * masked_bilateral_filter   gaustudio/scripts/extract_pcd.py:185-238   (cv2.dilate + cv2.bilateralFilter,
    OpenCV 4.13 float path: circular support of radius d/2, REFLECT_101 border, centre weight 1; OpenCV evaluates
    the range kernel through a 4096-bin interpolated table, this restatement evaluates it directly -- the
    difference is < 1e-5 of the depth range and is the tolerance of the golden test);
  * the per-view body of main()   extract_pcd.py:314-337   (mask, filter, depth2normal, -1 fill, world rotation,
    validity, negation);
  * normal_fusion   extract_pcd.py:108-183   (two weighted accumulation passes, consistency threshold 0.8,
    k=10 nearest-neighbour smoothing with exp(-dist/0.1)).
"""
import numpy as np

f32 = np.float32


def reflect101(i, n):
    """OpenCV's borderInterpolate for BORDER_REFLECT_101: reflect until the index is inside, 0 when n == 1."""
    i = np.asarray(i, np.int64)
    if n == 1:
        return np.zeros_like(i)
    while ((i < 0) | (i >= n)).any():
        i = np.where(i < 0, -i, np.where(i >= n, 2 * n - 2 - i, i))
    return i


def masked_bilateral_filter(depth, mask, d=3, sigma_color=75.0, sigma_space=75.0):
    depth = np.asarray(depth, f32)
    mask = np.asarray(mask).astype(bool)
    H, W = depth.shape
    r = d // 2
    assert d % 2 == 1 and d >= 1
    # cv2.dilate of the invalid mask with a d x d box; pixels outside the image never make a window invalid
    inv = ~mask
    dil = np.zeros_like(inv)
    for dy in range(-r, r + 1):
        for dx in range(-r, r + 1):
            if abs(dy) >= H or abs(dx) >= W:  # the shifted window lies wholly outside the image
                continue
            ys, ye = max(0, -dy), min(H, H - dy)
            xs, xe = max(0, -dx), min(W, W - dx)
            dil[ys:ye, xs:xe] |= inv[ys + dy:ye + dy, xs + dx:xe + dx]
    new_mask = ~dil
    valid = new_mask & ~np.isnan(depth)
    out = depth.copy()
    if not valid.any():
        return out, new_mask
    vmin = depth[valid].min()
    vmax = depth[valid].max()
    rng = f32(vmax - vmin)
    with np.errstate(invalid="ignore", divide="ignore"):
        norm = ((depth - vmin) / rng).astype(f32)
    norm[~valid] = 0
    # cv2.bilateralFilter, 32F: radius = d/2, support r_ij <= radius, border REFLECT_101
    gc = -0.5 / (float(sigma_color) ** 2)
    gs = -0.5 / (float(sigma_space) ** 2)
    pad = norm[np.ix_(reflect101(np.arange(-r, H + r), H), reflect101(np.arange(-r, W + r), W))]
    num = norm.astype(np.float64).copy()
    den = np.ones((H, W), np.float64)
    if float(norm.max()) - float(norm.min()) >= np.finfo(f32).eps:  # OpenCV copies a constant image through
        for dy in range(-r, r + 1):
            for dx in range(-r, r + 1):
                rr = np.sqrt(float(dy * dy + dx * dx))
                if rr > r or (dy == 0 and dx == 0):
                    continue
                nb = pad[r + dy:r + dy + H, r + dx:r + dx + W]
                diff = np.abs(nb - norm).astype(np.float64)
                w = np.float32(np.exp(rr * rr * gs)) * np.exp(diff * diff * gc)
                num += nb * w
                den += w
    filt = (num / den).astype(f32)
    den_out = (filt * rng).astype(f32) + vmin
    out[valid] = den_out[valid]
    return out, new_mask


def depth2normal_camera(depth, fx, fy, cx, cy, d_min=1e-3, d_max=100000.0):
    """Camera.depth2normal(coordinate='camera') -- gaustudio/datasets/__init__.py:342-380 (k = 3)."""
    depth = np.asarray(depth, f32)
    H, W = depth.shape
    u = (np.arange(W, dtype=f32) / f32(W - 1)) * f32(W - 1)
    v = (np.arange(H, dtype=f32) / f32(H - 1)) * f32(H - 1)
    ifx, ify, ox, oy = f32(1.0) / f32(fx), f32(1.0) / f32(fy), f32(-cx) / f32(fx), f32(-cy) / f32(fy)
    X = (u[None, :] * depth) * ifx + depth * ox
    Y = (v[:, None] * depth) * ify + depth * oy
    P = np.stack([X, Y, depth], -1).astype(f32)
    Pp = np.pad(P, ((1, 1), (1, 1), (0, 0)))
    ok = (Pp[..., 2] > d_min) & (Pp[..., 2] < d_max)
    vert = Pp[:-2, 1:-1] - Pp[2:, 1:-1]
    hori = Pp[1:-1, :-2] - Pp[1:-1, 2:]
    vm = ok[1:-1, 1:-1] & ok[:-2, 1:-1] & ok[2:, 1:-1] & ok[1:-1, :-2] & ok[1:-1, 2:]
    n = -np.cross(vert, hori)
    n = n / np.maximum(np.linalg.norm(n, axis=-1, keepdims=True), 1e-12)
    n = n.astype(f32)
    n[~vm] = -1
    return n


def view_normals(filtered, fg, opacity, median_depth, median_id, fx, fy, cx, cy, extrinsics, scene_radius):
    """extract_pcd.py:325-335 for one view, given the filtered depth and the dilated mask."""
    opacity = np.asarray(opacity, f32)
    cam_n = depth2normal_camera(filtered, fx, fy, cx, cy)
    cam_n[~np.asarray(fg, bool)] = -1
    E = np.asarray(extrinsics, f32)
    rot = np.linalg.inv(E[:3, :3]).T.astype(f32)  # normal2worldnormal, datasets/__init__.py:382-388
    world = (cam_n.reshape(-1, 3) @ rot).reshape(cam_n.shape).astype(f32)
    valid = (np.asarray(median_depth, f32) < f32(scene_radius * 0.8)) & (opacity > f32(0.5))
    wsum = (world[..., 0] + world[..., 1]) + world[..., 2]
    valid = (wsum > -3) & valid
    return {"cam_normals": cam_n, "valid": valid, "world_sum": wsum,
            "ids": np.asarray(median_id)[valid].astype(np.int64), "normals": (-world[valid]).astype(f32),
            "conf": opacity[valid]}


def extract_view(depth, opacity, median_depth, median_id, fx, fy, cx, cy, extrinsics, scene_radius, d=3,
                 sigma_color=75.0, sigma_space=75.0):
    """extract_pcd.py:314-337 for one view."""
    fg = np.asarray(opacity, f32) > f32(0.1)
    filtered, fg = masked_bilateral_filter(depth, fg, d, sigma_color, sigma_space)
    out = view_normals(filtered, fg, opacity, median_depth, median_id, fx, fy, cx, cy, extrinsics, scene_radius)
    out.update(filtered=filtered, fg_mask=fg)
    return out


def _pass_weights(xyz, cam_t, ids, normals, conf):
    v = cam_t[None, :].astype(f32) - xyz[ids]
    dist = np.linalg.norm(v, axis=1).astype(f32)
    vd = v / dist[:, None]
    vw = np.abs((vd * normals).sum(1))
    return (conf * vw * (f32(1.0) / (dist + f32(1e-6)))).astype(f32)


def fusion_pass(xyz, ids_list, normals_list, conf_list, cam_ts, mean=None, thresh=0.8):
    """One accumulation pass of normal_fusion (extract_pcd.py:117-136 / :143-165), dense over Gaussian ids.
    Returns (sum_normals [P,3] f64, sum_weights [P] f64, touched [P] bool)."""
    P = xyz.shape[0]
    sn = np.zeros((P, 3), np.float64); sw = np.zeros(P, np.float64); touched = np.zeros(P, bool)
    for ids, n, c, t in zip(ids_list, normals_list, conf_list, cam_ts):
        w = _pass_weights(xyz, np.asarray(t, f32), ids, n, c)
        touched[ids] = True
        if mean is not None:
            keep = np.linalg.norm(n - mean[ids], axis=1) < thresh
            ids, n, w = ids[keep], n[keep], w[keep]
        np.add.at(sn, ids, n * w[:, None]); np.add.at(sw, ids, w)
    return sn, sw, touched


def _mean(sn, sw):
    with np.errstate(invalid="ignore", divide="ignore"):
        m = (sn / sw[:, None]).astype(f32)
    return m / np.maximum(np.linalg.norm(m, axis=1, keepdims=True), 1e-12)


def normal_fusion(xyz, ids_list, normals_list, conf_list, cam_ts, smooth=True, k=10, sigma=0.1):
    """extract_pcd.py:108-183.  cam_ts: per view `extrinsics[:3, 3]` (what the reference uses as the camera position).
    Returns (unique_ids int64 ascending, normals [n,3])."""
    xyz = np.asarray(xyz, f32)
    sn, sw, touched = fusion_pass(xyz, ids_list, normals_list, conf_list, cam_ts)
    mean = _mean(sn, sw)
    sn, sw, _ = fusion_pass(xyz, ids_list, normals_list, conf_list, cam_ts, mean=mean)
    mean = _mean(sn, sw)
    uid = np.nonzero(touched)[0].astype(np.int64)
    mean = mean[uid]
    if not smooth:
        return uid, mean.astype(f32)
    from scipy.spatial import cKDTree
    pts = xyz[uid]
    dist, idx = cKDTree(pts).query(pts, k=k)
    w = np.exp(-dist / sigma)
    sm = (mean[idx].astype(np.float64) * w[..., None]).sum(1).astype(f32)
    sm = sm / np.maximum(np.linalg.norm(sm, axis=1, keepdims=True), 1e-12)
    return uid, sm.astype(f32)
