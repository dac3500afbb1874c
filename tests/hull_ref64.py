"""Restatements of the VisualHull and depth initializers (DESIGN.md 7k), shared by the CPU and GPU tests:

  linspace64(r, res)                 np.linspace(-r, r, res) as i step + start, the last node r
  grid_points(res, r, t)             the reference's float32 grid: meshgrid(lin, lin, lin) - t, node (i res + j) res + k
  inside64(x, P, W, H, mask)         insideView in float64 from float32 x and P, plus a flag where float32 evaluation
                                     can decide otherwise (a derived bound; see below)
  carve64(x, cams)                   occupancy and flags over cameras (P, W, H, mask | None)
  inside_view32(x, P, W, H, mask)    the reference's Camera.insideView loop step in float32 torch (mask.py:59-68)
  carve32(x, cams)                   the reference's per-camera loop with it
  hull_mesh64(occ, threshold, r, t)  marching cubes of the occupancy, world vertices in double rounded once
  depth_chain(views)                 DepthInitializer's float16 chain in numpy (depth.py:37-90)

Every function takes torch tensors on any device (the float64 work runs where the tensors are) or numpy arrays.

The flag bound.  The reference forms clip = [x 1] P in float32: any summation order of the four products is within
gamma_4 S_j of the exact value, S_j = sum_i |v_i P_ij|; we take e_j = 5u S_j (u = 2^-24), which also covers this
restatement's own double rounding.  A node is flagged for a camera when
  |clip_z| <= e_z                                            (the clip_z > 0 decision)
  |clip_w| <= e_w                                            (ndc itself is undetermined)
  ||ndc_x| - 1| <= E_x or ||ndc_y| - 1| <= E_y               (the range decisions), with
      E = (e_xy + |ndc| e_w) / (|clip_w| - e_w) + u |ndc|   the float32 error of the division's result
  the mask differs among the pixels (trunc(p +- E_p)) with E_p = W/2 E + 4u W   (integer pixel edges, the clamp)
"""
import numpy as np
import torch

import sap_ref64

U32 = 2.0 ** -24


def linspace64(r, res):
    start, stop = -float(r), float(r)
    step = (stop - start) / (res - 1)
    lin = np.arange(res, dtype=np.float64) * step + start
    lin[-1] = stop
    return lin


def grid_points(res, r, t, device="cpu"):
    """-> float32 [res^3, 3] on device: node (i res + j) res + k at (lin[j], lin[i], lin[k]) - t."""
    lin = torch.from_numpy(linspace64(r, res)).to(device)
    t = torch.as_tensor(np.asarray(t, np.float64), device=device)
    i, j, k = torch.meshgrid(lin, lin, lin, indexing="ij")
    return torch.stack([j - t[0], i - t[1], k - t[2]], -1).reshape(-1, 3).float()


def _t(a, device):
    return a.to(device) if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a)).to(device)


def inside64(x, P, W, H, mask=None):
    """x float32 [N,3], P float32 [4,4] (row-vector clip = [x 1] P) -> (inside bool [N], flag bool [N]), float64."""
    x = _t(x, None)
    dev = x.device
    xd = x.double()
    Pd = _t(P, dev).double()
    clip, S = [], []
    for c in range(4):
        clip.append(((xd[:, 0] * Pd[0, c] + xd[:, 1] * Pd[1, c]) + xd[:, 2] * Pd[2, c]) + Pd[3, c])
        S.append((xd.abs() * Pd[:3, c].abs()).sum(1) + Pd[3, c].abs())
    cx, cy, cz, cw = clip
    e = [5 * U32 * s for s in S]
    nx, ny = cx / cw, cy / cw
    valid = (cz > 0) & (nx >= -1) & (nx <= 1) & (ny >= -1) & (ny <= 1)
    px = ((nx + 1) * 0.5 * W).nan_to_num(0.0, 0.0, 0.0).clamp(0, W).long().clamp(max=W - 1)
    py = ((ny + 1) * 0.5 * H).nan_to_num(0.0, 0.0, 0.0).clamp(0, H).long().clamp(max=H - 1)
    m = None if mask is None else (_t(mask, dev) != 0)
    inside = valid.clone()
    if m is not None:
        inside &= m[py, px]
    # flags
    aw = cw.abs()
    undetermined = aw <= e[3]
    den = (aw - e[3]).clamp_min(1e-300)
    Ex = (e[0] + nx.abs() * e[3]) / den + U32 * nx.abs()
    Ey = (e[1] + ny.abs() * e[3]) / den + U32 * ny.abs()
    flag = (cz.abs() <= e[2]) | undetermined
    flag |= ((nx.abs() - 1).abs() <= Ex) | ((ny.abs() - 1).abs() <= Ey)
    if m is not None:
        Epx, Epy = W / 2 * Ex + 4 * U32 * W, H / 2 * Ey + 4 * U32 * H
        pxf, pyf = (nx + 1) * 0.5 * W, (ny + 1) * 0.5 * H
        cand = lambda p, E, n: [(p + s * E).nan_to_num(0.0, 0.0, 0.0).clamp(0, n).long().clamp(max=n - 1)
                                for s in (-1, 1)]
        xs, ys = cand(pxf, Epx, W), cand(pyf, Epy, H)
        vals = torch.stack([m[yy, xx] for yy in ys for xx in xs])
        flag |= valid & (vals.any(0) != vals.all(0))
    return inside, flag


def carve64(x, cams, chunk=1 << 22):
    """cams: [(P, W, H, mask | None)] -> (occ bool [N], flagged bool [N]) over every camera (a node is flagged when any
    camera's decision for it is within the bound)."""
    x = _t(x, None)
    occ = torch.ones(x.shape[0], dtype=torch.bool, device=x.device)
    flag = torch.zeros_like(occ)
    for s in range(0, x.shape[0], chunk):
        xs = x[s:s + chunk]
        for P, W, H, m in cams:
            ins, fl = inside64(xs, P, W, H, m)
            occ[s:s + chunk] &= ins
            flag[s:s + chunk] |= fl
    return occ, flag


def inside_view32(x, P, W, H, mask=None):
    """Camera.insideView of the reference (datasets/__init__.py:268-305), restated op for op in float32 torch."""
    if mask is None:
        mask = torch.ones(H, W, device=x.device)
    h = torch.cat([x, torch.ones_like(x[:, :1])], dim=-1)
    clip = torch.matmul(h, P)
    ndc = clip[:, :3] / clip[:, 3:4]
    pixel_x = (ndc[:, 0] + 1) * 0.5 * W
    pixel_y = (1 + ndc[:, 1]) * 0.5 * H
    valid = (clip[:, 2] > 0) & (ndc[:, 0] >= -1) & (ndc[:, 0] <= 1) & (ndc[:, 1] >= -1) & (ndc[:, 1] <= 1)
    inside = torch.zeros_like(valid, dtype=torch.bool)
    if valid.any():
        vx = pixel_x[valid].long().clamp(0, W - 1)
        vy = pixel_y[valid].long().clamp(0, H - 1)
        inside[valid] = mask[vy, vx].bool()
    return inside


def carve32(x, cams):
    """mask.py:57-68: filled &= insideView(points[inside_view_idx], mask) scattered back, camera by camera."""
    filled = torch.ones(x.shape[0], dtype=torch.bool, device=x.device)
    for P, W, H, m in cams:
        P = _t(P, x.device).float()
        iv = inside_view32(x, P, W, H)
        idx = torch.where(iv)[0]
        cam = torch.zeros_like(filled)
        cam[idx] = inside_view32(x[idx], P, W, H, None if m is None else _t(m, x.device))
        filled &= cam
    return filled


def hull_mesh64(occ, threshold, r, t):
    """-> (vertices float32 [V,3], faces int64 [F,3], vertices float64 before rounding) in gsr_hull_marching_cubes'
    order: the project's marching cubes of the empty side (sap_ref64.marching_cubes64 on +-1), each vertex placed at
    the threshold from its empty end, the first two axes swapped and each triangle reversed."""
    occ = np.asarray(occ.cpu() if isinstance(occ, torch.Tensor) else occ).astype(bool)
    res = occ.shape[0]
    v, f = sap_ref64.marching_cubes64(np.where(occ, -1.0, 1.0))
    axis = np.argmax(v != np.floor(v), axis=1)  # the one coordinate at a half-integer
    c = np.floor(v).astype(np.int64)
    n0 = occ[c[:, 0], c[:, 1], c[:, 2]]
    frac = np.where(n0, 1.0 - threshold, threshold)
    q = c.astype(np.float64)
    q[np.arange(len(q)), axis] += frac
    t = np.asarray(t, np.float64)
    world = lambda qa, ta: ((qa / (res - 1)) * (2.0 * r) - r) - ta
    w = np.stack([world(q[:, 1], t[0]), world(q[:, 0], t[1]), world(q[:, 2], t[2])], 1)
    return w.astype(np.float32), f[:, ::-1].copy(), w


def signed_volume(v, f):
    v = np.asarray(v, np.float64)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    return float(np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6.0)


def depth_chain(views):
    """views: [(world xyz [h,w,3] float32, image [h,w,3] float32, depth [h,w] float32, fx, fy float32)] ->
    dict(points16, colors uint8, scales16, xyz, rgb, log_scale [N,3], opacity) as depth.py stores and builds them."""
    rows = []
    for xyz, img, depth, fx, fy in views:
        scale = depth / ((np.float32(fx) + np.float32(fy)) / np.float32(2))
        rows.append(np.hstack((xyz.reshape(-1, 3), img.reshape(-1, 3), scale.reshape(-1, 1))).astype(np.float16))
    pcd = np.concatenate(rows)
    points16, scales16 = pcd[:, :3], np.ascontiguousarray(pcd[:, 6:])  # as read back from scales.bin
    colors = (pcd[:, 3:6] * 255).astype(np.uint8)
    with np.errstate(divide="ignore", invalid="ignore"):
        log_scale = np.repeat(np.log(scales16), 3, axis=1).astype(np.float32)
    return dict(points16=points16, colors=colors, scales16=scales16.reshape(-1),
                xyz=points16.astype(np.float64).astype(np.float32),
                rgb=(torch.from_numpy(colors).float() / 255.0).numpy(), log_scale=log_scale,
                opacity=np.zeros((len(pcd), 1), np.float32))

