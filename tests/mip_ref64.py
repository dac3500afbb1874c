"""Float64 reference of the Mip-Splatting projection and of the 3D smoothing filter (torch / numpy, CPU).

Projection: proj_ref64's projection with the 2D Mip filter in place of the 0.3 dilation (include/gsr.h,
gsr_forward_mip).  With (a, b, c) the undilated cov2D and k = kernel_size:
    det0 = max(1e-6, ac - b^2), det1 = max(1e-6, (a+k)(c+k) - b^2), coef = sqrt(det0 / (det1 + 1e-6) + 1e-6),
    coef = 0 when either clamp fired (no gradient there);  cov' = (a+k, b, c+k) -> conic, radius, rect;  o' = o coef.
Everything else (means2D, depth, colour, lateral clamp, regularised conic backward, scale-gradient convention) is
proj_ref64's, reused through its differentiable `_state`: the undilated cov2D is its cov2D minus 0.3 (exact to float64
rounding).  Un-fused inputs only, like the Mip entry points.

3D filter: `filter3d` restates MipPointCloud.compute_3D_filter (gsr_mip_filter3d) vectorised over cameras, in float64.
"""
import math

import numpy as np
import torch

import proj_ref64 as R

F64 = torch.float64
EPS6 = 1e-6
TILE = R.TILE


def mip_state(p, cam, k, clamped=None, sh_dir_grad=True):
    """Differentiable per-Gaussian Mip projection of the float64 tensors in `p` (un-fused keys)."""
    s = R._state(p, cam, False, clamped=clamped, sh_dir_grad=sh_dir_grad)
    a = s["cov2D"][:, 0] - 0.3
    b = s["cov2D"][:, 1]
    c = s["cov2D"][:, 2] - 0.3
    d0 = a * c - b * b
    d1 = (a + k) * (c + k) - b * b
    fired = ((d0 <= EPS6) | (d1 <= EPS6)).detach()
    d0c, d1c = torch.where(fired, torch.ones_like(d0), d0), torch.where(fired, torch.ones_like(d1), d1)
    coef = torch.where(fired, torch.zeros_like(d0), torch.sqrt(d0c / (d1c + EPS6) + EPS6))
    ap, cp = a + k, c + k
    conA, conB, conC = R._Conic.apply(ap, b, cp)
    return dict(s, conic=torch.stack([conA, conB, conC], 1), cov2D=torch.stack([ap, b, cp], 1), coef=coef,
                det0=d0, det1=d1, opacity=s["opacity"] * coef)


def forward(p, cam, k):
    """Float64 forward of every Gaussian: means2D, conic, opacity (o'), coef, depth, rgb, clamped, radius (0 where
    culled), the tile rect (x0, y0, x1, y1), the undilated dets det0 / det1 and txtz_over_lim."""
    q = R._params(p, False)
    with torch.no_grad():
        s = mip_state(q, cam, k)
        W, H = cam["W"], cam["H"]
        a, b, c = s["cov2D"].unbind(1)
        det = a * c - b * b
        mid = 0.5 * (a + c)
        sq = torch.sqrt(torch.clamp(mid * mid - det, min=0.1))
        radius = torch.ceil(3 * torch.sqrt(torch.maximum(mid + sq, mid - sq)))
        gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
        px, py = s["means2D"].unbind(1)
        ri = torch.nan_to_num(radius, nan=0.0, posinf=0.0).to(torch.int64)
        rect = lambda v, lo: torch.clamp(torch.trunc(v), min=0).clamp(max=lo).to(torch.int64)
        x0, x1 = rect((px - ri) / TILE, gx), rect((px + ri + TILE - 1) / TILE, gx)
        y0, y1 = rect((py - ri) / TILE, gy), rect((py + ri + TILE - 1) / TILE, gy)
        vis = (s["depth"] > 0.2) & (det != 0) & ((x1 - x0) * (y1 - y0) != 0)
        # the value under the ceil: integer outputs are only pinned away from its jumps
        pre_ceil = 3 * torch.sqrt(torch.maximum(mid + sq, mid - sq))
    return dict(means2D=s["means2D"], conic=s["conic"], opacity=s["opacity"], coef=s["coef"], depth=s["depth"],
                rgb=s["color_raw"].clamp_min(0), clamped=s["color_raw"] < 0, cov2D=s["cov2D"],
                radius=torch.where(vis, ri, torch.zeros_like(ri)), rect=torch.stack([x0, y0, x1, y1], 1), vis=vis,
                pre_ceil=pre_ceil, det0=s["det0"], det1=s["det1"], txtz_over_lim=s["txtz_over_lim"])


def upstream_from_sums(sums, p, cam, k, radii):
    """The accumulator [P,12] -> upstream dict, as proj_ref64.upstream_from_sums but with the Mip conic (the one the
    splats carry).  `opacity` is dL/do'."""
    S = R.t64(sums)
    P = S.shape[0]
    live = torch.as_tensor(np.asarray(radii)).reshape(-1) > 0
    S = torch.where(live[:, None], S, torch.zeros_like(S))
    q = R._params(p, False)
    con = torch.zeros(P, 3, dtype=F64)
    idx = live.nonzero().reshape(-1)
    if idx.numel():
        with torch.no_grad():
            con[idx] = mip_state({kk: (v[idx] if v is not None else None) for kk, v in q.items()}, cam, k)["conic"]
    A, B, C = con.unbind(1)
    Sx, Sy = S[:, 5], S[:, 6]
    m2 = torch.stack([-(A * Sx + B * Sy) * (0.5 * cam["W"]), -(C * Sy + B * Sx) * (0.5 * cam["H"]),
                      torch.zeros(P, dtype=F64)], 1)
    return dict(mean2D=m2, conic=-0.5 * S[:, 7:10], color=S[:, 0:3].clone(), depth=S[:, 3].clone(),
                opacity=S[:, 4].clone())


def vjp(p, cam, k, upstream, radii, clamped=None):
    """Gradients of every input of the Mip projection, keyed like proj_ref64.vjp (un-fused); `opacity` is the gradient
    w.r.t. the input opacity (dL/do' coef), and the opacity upstream also reaches cov3D, scales, rotations and means
    through coef."""
    q = R._params(p, False)
    P = q["means3D"].shape[0]
    up = {kk: R.t64(v) for kk, v in upstream.items()}
    live = torch.as_tensor(np.asarray(radii)).reshape(-1) > 0
    idx = live.nonzero().reshape(-1)
    keys = [kk for kk, v in q.items() if v is not None]
    full = {kk: torch.zeros_like(q[kk]) for kk in keys}
    full["cov3D"] = torch.zeros(P, 6, dtype=F64)
    if idx.numel():
        leaves = {kk: q[kk][idx].clone().requires_grad_(True) for kk in keys}
        cm = None if clamped is None else np.asarray(clamped).reshape(P, 3)[idx.numpy()].astype(bool)
        s = mip_state(leaves, cam, k, clamped=cm)
        u = {kk: v[idx] for kk, v in up.items()}
        L = ((u["mean2D"][:, :2] * s["ndc"]).sum() + (u["conic"][:, 0] * s["conic"][:, 0]).sum()
             + (2 * u["conic"][:, 1] * s["conic"][:, 1]).sum() + (u["conic"][:, 2] * s["conic"][:, 2]).sum()
             + (u["color"] * s["rgb"]).sum() + (u["depth"] * s["depth"]).sum() + (u["opacity"] * s["opacity"]).sum())
        ins = [leaves[kk] for kk in keys] + [s["cov3D"]]
        gs = torch.autograd.grad(L, ins, allow_unused=True)
        for kk, g in zip(keys + ["cov3D"], gs):
            if g is not None:
                full[kk][idx] = g
    if "scales" in full:
        full["scales"] = full["scales"] / cam["mod"]
    zero = lambda x: torch.where(live.reshape((-1,) + (1,) * (x.dim() - 1)), x, torch.zeros_like(x))
    m2 = zero(up["mean2D"]).clone()
    m2[:, 2] = 0
    con = zero(up["conic"])
    out = dict(full, mean2D=m2, conic=torch.stack([con[:, 0], con[:, 1], torch.zeros(P, dtype=F64), con[:, 2]], 1),
               color=zero(up["color"]), depth=zero(up["depth"]))
    out["opacity"] = full.pop("opacities")
    del out["opacities"]
    return out


# ---- 3D smoothing filter ------------------------------------------------------------------------------------------
def camera_records(cameras):
    """[C,16] float64: R (row-major Camera.R), T, fx, fy, W, H -- the records of gsr_mip_filter3d."""
    rows = []
    for c in cameras:
        fx = c.image_width / (2.0 * math.tan(c.FoVx * 0.5))
        fy = c.image_height / (2.0 * math.tan(c.FoVy * 0.5))
        rows.append(np.concatenate([np.asarray(c.R, np.float64).reshape(9), np.asarray(c.T, np.float64).reshape(3),
                                    [fx, fy, c.image_width, c.image_height]]))
    return np.stack(rows)


def filter3d_terms(xyz, recs):
    """Per (Gaussian, camera): p.z, u, v and visibility, in float64.  xyz [P,3], recs [C,16]."""
    x = np.asarray(xyz, np.float64)
    Rm = recs[:, :9].reshape(-1, 3, 3)
    p = np.einsum("pi,cij->cpj", x, Rm) + recs[:, None, 9:12]
    z = np.maximum(p[..., 2], 0.001)
    W, H = recs[:, 14:15], recs[:, 15:16]
    u = p[..., 0] / z * recs[:, 12:13] + W / 2
    v = p[..., 1] / z * recs[:, 13:14] + H / 2
    seen = (p[..., 2] > 0.2) & (u >= -0.15 * W) & (u <= 1.15 * W) & (v >= -0.15 * H) & (v <= 1.15 * H)
    return p[..., 2], u, v, seen


def filter3d(xyz, recs):
    """-> (filter_3D [P] float64, seen [P] bool).  Raises ValueError when no Gaussian is seen."""
    pz, _, _, seen = filter3d_terms(xyz, recs)
    d = np.where(seen, pz, np.inf).min(axis=0)
    d = np.minimum(d, 100000.0)
    any_seen = seen.any(axis=0)
    if not any_seen.any():
        raise ValueError("no camera sees any Gaussian")
    d = np.where(any_seen, d, d[any_seen].max())
    return d / recs[:, 12].max() * math.sqrt(0.2), any_seen


def near_boundary(xyz, recs, rel=1e-5):
    """[P] bool: some camera's visibility test of the Gaussian lies within `rel` (relative) of one of its thresholds."""
    pz, u, v, _ = filter3d_terms(xyz, recs)
    W, H = recs[:, 14:15], recs[:, 15:16]
    close = lambda a, t: np.abs(a - t) <= rel * np.maximum(np.abs(t), 1.0)
    near = close(pz, 0.2) | close(u, -0.15 * W) | close(u, 1.15 * W) | close(v, -0.15 * H) | close(v, 1.15 * H)
    return near.any(axis=0)
