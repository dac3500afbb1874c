"""Float64 restatements of the Gaussian initializers (gaustudio/pipelines/initializers/{pcd,mesh}.py and simple_knn's
distCUDA2) for tests/test_init_cpu.py and tests/test_gpu_init.py:

  tribox64 / tribox_exact     Akenine-Moller's tribox3 in float64 (its op order), and an exact separating-axis test
                              in fractions.Fraction (a touch overlaps)
  occupied64                  the occupied cells of open3d's CreateFromTriangleMeshWithinBounds, by brute force over
                              each triangle's bounding box
  closest_bary64 / closest_brute   the kernel's closest point (barycentrics), and brute force over vertices, edges
                              and the face interior
  candidates64                the kernel's candidate cells of one triangle (columns along the dominant normal axis)
  vertex_normals64            open3d's compute_vertex_normals, a per-face loop
  normal2rotation64 / normal2rotation_torch32   pcd.py:12-37 in float64, and the reference's float32 torch code
  sugar64                     mesh.py's placement (positions, normals, colours, scales), per-face loops
  dist2_64                    mean of the 3 smallest squared distances to other points (cKDTree k=4)
"""
from fractions import Fraction

import numpy as np

SH_C0 = 0.28209479177387814
BARY = {1: [[1 / 3, 1 / 3, 1 / 3]],
        3: [[1 / 2, 1 / 4, 1 / 4], [1 / 4, 1 / 2, 1 / 4], [1 / 4, 1 / 4, 1 / 2]],
        4: [[1 / 3, 1 / 3, 1 / 3], [2 / 3, 1 / 6, 1 / 6], [1 / 6, 2 / 3, 1 / 6], [1 / 6, 1 / 6, 2 / 3]],
        6: [[2 / 3, 1 / 6, 1 / 6], [1 / 6, 2 / 3, 1 / 6], [1 / 6, 1 / 6, 2 / 3], [1 / 6, 5 / 12, 5 / 12],
            [5 / 12, 1 / 6, 5 / 12], [5 / 12, 5 / 12, 1 / 6]]}
RADIUS = {1: 1. / 2. / np.sqrt(3.), 3: 1. / 2. / (np.sqrt(3.) + 1.), 4: 1 / (4. * np.sqrt(3.)),
          6: 1 / (4. + 2. * np.sqrt(3.))}


# ---- tribox3 ----
def tribox64(c, h, t):
    """tribox3 in float64, vectorised: c [N,3] box centres, h half-size, t [N,3,3] triangles -> bool [N]."""
    c, t = np.asarray(c, np.float64), np.asarray(t, np.float64)
    v0, v1, v2 = t[:, 0] - c, t[:, 1] - c, t[:, 2] - c
    e0, e1, e2 = v1 - v0, v2 - v1, v0 - v2
    X, Y, Z = 0, 1, 2
    sep = np.zeros(len(c), bool)

    def axis(pa, pb, fa, fb):
        mn, mx = np.minimum(pa, pb), np.maximum(pa, pb)
        rad = fa * h + fb * h
        return (mn > rad) | (mx < -rad)

    for e, (p, q), (r, s), (u, w) in ((e0, (v0, v2), (v0, v2), (v1, v2)), (e1, (v0, v2), (v0, v2), (v0, v1)),
                                      (e2, (v0, v1), (v0, v1), (v1, v2))):
        fex, fey, fez = np.abs(e[:, X]), np.abs(e[:, Y]), np.abs(e[:, Z])
        sep |= axis(e[:, Z] * p[:, Y] - e[:, Y] * p[:, Z], e[:, Z] * q[:, Y] - e[:, Y] * q[:, Z], fez, fey)
        sep |= axis(-e[:, Z] * r[:, X] + e[:, X] * r[:, Z], -e[:, Z] * s[:, X] + e[:, X] * s[:, Z], fez, fex)
        sep |= axis(e[:, Y] * u[:, X] - e[:, X] * u[:, Y], e[:, Y] * w[:, X] - e[:, X] * w[:, Y], fey, fex)
    for d in range(3):
        mn = np.minimum(np.minimum(v0[:, d], v1[:, d]), v2[:, d])
        mx = np.maximum(np.maximum(v0[:, d], v1[:, d]), v2[:, d])
        sep |= (mn > h) | (mx < -h)
    n = np.stack([e0[:, Y] * e1[:, Z] - e0[:, Z] * e1[:, Y], e0[:, Z] * e1[:, X] - e0[:, X] * e1[:, Z],
                  e0[:, X] * e1[:, Y] - e0[:, Y] * e1[:, X]], 1)
    pos = n > 0
    vmin = np.where(pos, -h - v0, h - v0)
    vmax = np.where(pos, h - v0, -h - v0)
    dmin = n[:, 0] * vmin[:, 0] + n[:, 1] * vmin[:, 1] + n[:, 2] * vmin[:, 2]
    dmax = n[:, 0] * vmax[:, 0] + n[:, 1] * vmax[:, 1] + n[:, 2] * vmax[:, 2]
    return ~sep & ~(dmin > 0) & (dmax >= 0)


def tribox_exact(c, h, t):
    """Exact separating-axis test in Fraction: the closed triangle and the closed box meet (a touch overlaps)."""
    F = lambda x: Fraction(float(x))
    c = [F(x) for x in c]
    h = F(h)
    v = [[F(t[i][d]) - c[d] for d in range(3)] for i in range(3)]
    e = [[v[(i + 1) % 3][d] - v[i][d] for d in range(3)] for i in range(3)]
    cross = lambda a, b: [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]
    axes = [[1, 0, 0], [0, 1, 0], [0, 0, 1], cross(e[0], e[1])]
    axes += [cross(ei, a) for ei in e for a in ([1, 0, 0], [0, 1, 0], [0, 0, 1])]
    for a in axes:
        if all(x == 0 for x in a):
            continue
        p = [sum(a[d] * vi[d] for d in range(3)) for vi in v]
        r = h * sum(abs(x) for x in a)
        if min(p) > r or max(p) < -r:
            return False
    return True


def box_centres(ijk, vs):
    """(-0.5 + idx vs) + vs / 2, left to right, per axis."""
    return (-0.5 + np.asarray(ijk, np.float64) * vs) + vs / 2


def voxel_centres(ijk, vs):
    """open3d's GetVoxelCenterCoordinate: (idx + 0.5) vs + origin, origin -0.5."""
    return (np.asarray(ijk, np.float64) + 0.5) * vs + -0.5


def _cell(x, vs, res):
    return int(min(max(np.floor((x - -0.5) / vs), -1.0), float(res)))


def candidates64(t, res, vs):
    """The cells k_vox_columns / k_vox_hits test for triangle t [3,3] (float64, normalised): per column of the grown
    bounding box along the two axes other than the normal's dominant one, the plane's slab grown by the rounding
    slack and one cell -> set of (i, j, k)."""
    t = np.asarray(t, np.float64)
    lo = [max(_cell(t[:, d].min(), vs, res) - 1, 0) for d in range(3)]
    hi = [min(_cell(t[:, d].max(), vs, res) + 1, res - 1) for d in range(3)]
    e, g = t[1] - t[0], t[2] - t[0]
    n = np.array([e[1] * g[2] - e[2] * g[1], e[2] * g[0] - e[0] * g[2], e[0] * g[1] - e[1] * g[0]])
    an = np.abs(n)
    a = (0 if an[0] >= an[2] else 2) if an[0] >= an[1] else (1 if an[1] >= an[2] else 2)
    u, w = (a + 1) % 3, (a + 2) % 3
    le, lg = np.sqrt(e @ e), np.sqrt(g @ g)
    with np.errstate(divide="ignore", invalid="ignore"):
        slack = 64.0 * 2.0 ** -53 * le * lg * (le + lg) / an[a]
    out = set()
    for iu in range(lo[u], hi[u] + 1):
        for iw in range(lo[w], hi[w] + 1):
            k0, k1 = lo[a], hi[a]
            if slack < 1.0:
                z = [t[0, a] - (n[u] * (-0.5 + (iu + (c & 1)) * vs - t[0, u]) +
                                n[w] * (-0.5 + (iw + (c >> 1)) * vs - t[0, w])) / n[a] for c in range(4)]
                k0 = max(k0, _cell(min(z) - slack, vs, 1 << 30) - 1)
                k1 = min(k1, _cell(max(z) + slack, vs, 1 << 30) + 1)
            for ka in range(k0, k1 + 1):
                c = [0, 0, 0]
                c[a], c[u], c[w] = ka, iu, iw
                out.add(tuple(c))
    return out


def occupied64(verts, faces, res, vs, chunk=1 << 22):
    """Ascending linear indices (i res + j) res + k of the cells some triangle overlaps (tribox64), testing every cell
    of each triangle's bounding box grown by one cell."""
    verts, faces = np.asarray(verts, np.float64), np.asarray(faces, np.int64)
    out = []
    for f in faces:
        t = verts[f]
        lo = np.clip(np.floor((t.min(0) + 0.5) / vs).astype(int) - 1, 0, res - 1)
        hi = np.clip(np.floor((t.max(0) + 0.5) / vs).astype(int) + 1, 0, res - 1)
        g = np.stack(np.meshgrid(*[np.arange(lo[d], hi[d] + 1) for d in range(3)], indexing="ij"), -1).reshape(-1, 3)
        for s in range(0, len(g), chunk):
            gg = g[s:s + chunk]
            hit = tribox64(box_centres(gg, vs), vs / 2, np.broadcast_to(t, (len(gg), 3, 3)))
            gg = gg[hit]
            out.append((gg[:, 0] * res + gg[:, 1]) * res + gg[:, 2])
    return np.unique(np.concatenate(out)) if out else np.empty(0, np.int64)


# ---- closest point ----
def closest_bary64(p, a, b, c):
    """The kernel's closest point in float64, its op order -> (squared distance, barycentrics): the plane's foot when
    Ericson's va, vb, vc are >= 0 with a positive sum, then the clamped projections onto ab, bc, ca (a zero edge gives
    its vertex); the first smallest wins."""
    p, a, b, c = (np.asarray(x, np.float64) for x in (p, a, b, c))
    ab, ac, ap, bp, cp = b - a, c - a, p - a, p - b, p - c
    dot = lambda x, y: (x[0] * y[0] + x[1] * y[1]) + x[2] * y[2]
    d1, d2, d3, d4, d5, d6 = dot(ab, ap), dot(ac, ap), dot(ab, bp), dot(ac, bp), dot(ab, cp), dot(ac, cp)
    vc, vb, va = d1 * d4 - d3 * d2, d5 * d2 - d1 * d6, d3 * d6 - d5 * d4
    den = (va + vb) + vc
    best = (np.inf, np.array([1.0, 0.0, 0.0]))
    if den > 0 and va >= 0 and vb >= 0 and vc >= 0:
        v, w = vb / den, vc / den
        best = _at(p, a, b, c, (1.0 - v) - w, v, w)
    for x, y, ix, iy in ((a, b, 0, 1), (b, c, 1, 2), (c, a, 2, 0)):
        d = y - x
        L = dot(d, d)
        t = min(max(dot(p - x, d) / L, 0.0), 1.0) if L > 0 else 0.0
        bc = [0.0, 0.0, 0.0]
        bc[ix], bc[iy] = 1.0 - t, t
        cand = _at(p, a, b, c, *bc)
        if cand[0] < best[0]:
            best = cand
    return best


def _at(p, a, b, c, u, v, w):
    q = (u * a + v * b) + w * c
    e = p - q
    return float((e[0] * e[0] + e[1] * e[1]) + e[2] * e[2]), np.array([u, v, w])


def closest_brute(p, a, b, c):
    """Squared distance from p to the closed triangle: the least over its vertices, its edges (clamped projections)
    and, when the projection falls inside, the plane."""
    p, a, b, c = (np.asarray(x, np.float64) for x in (p, a, b, c))
    best = min(np.sum((p - x) ** 2) for x in (a, b, c))
    for x, y in ((a, b), (b, c), (c, a)):
        d = y - x
        L = d @ d
        if L > 0:
            s = np.clip((p - x) @ d / L, 0, 1)
            best = min(best, np.sum((p - (x + s * d)) ** 2))
    n = np.cross(b - a, c - a)
    nn = n @ n
    if nn > 0:
        q = p - ((p - a) @ n / nn) * n
        inside = all(np.cross(y - x, q - x) @ n >= 0 for x, y in ((a, b), (b, c), (c, a)))
        if inside:
            best = min(best, np.sum((p - q) ** 2))
    return float(best)


# ---- vertex normals, normal2rotation, SuGaR ----
def vertex_normals64(verts, faces):
    v = np.asarray(verts, np.float64)
    out = np.zeros_like(v)
    for f in np.asarray(faces):
        n = np.cross(v[f[1]] - v[f[0]], v[f[2]] - v[f[0]])
        for c in f:
            out[c] += n
    l = np.sqrt((out ** 2).sum(1, keepdims=True))
    return np.where(l > 0, out / np.where(l > 0, l, 1), 0.0)


def normal2rotation64(n):
    """pcd.py:12-37 in float64 -> (q [N,4], r [N], s [N] the norm of R0 before normalisation, R0, R1, n); the sign
    decisions of R0 and R1 are taken in float64."""
    n = np.asarray(n, np.float64)
    n = n / np.maximum(np.linalg.norm(n, axis=1, keepdims=True), 1e-12)
    R0 = np.array([1.0, 0, 0]) - n[:, :1] * n
    s = np.linalg.norm(R0, axis=1)
    R0 = R0 * np.sign(R0[:, :1])
    R0 = R0 / np.maximum(np.linalg.norm(R0, axis=1, keepdims=True), 1e-12)
    R1 = np.cross(n, R0)
    R1 = R1 * (np.sign(R1[:, 1:2]) * np.sign(n[:, 2:]))
    tr = R0[:, 0] + R1[:, 1] + n[:, 2] + 1e-6
    r = np.sqrt(1 + tr) / 2
    q = np.stack([r, (R1[:, 2] - n[:, 1]) / (4 * r), (n[:, 0] - R0[:, 2]) / (4 * r), (R0[:, 1] - R1[:, 0]) / (4 * r)], -1)
    return q, r, s, R0, R1, n


def quat_bound(q64, r, s):
    """Bound on |q32 - q64| per component.  R0 = w0 - n_x n has norm s = sqrt(1 - n_x^2) before it is normalised, so
    the float32 errors of R0 and R1 (a few eps) grow by 1/s.  r = sqrt(1 + tr) / 2 with tr a sum of four terms of
    size <= 1, so |d(1 + tr)| <= 16 eps / s and |dr| / r <= 16 eps / (8 r^2 s); q_k = x_k / 4r with |x_k| <= 2 and
    |dx_k| <= 8 eps / s.  Hence |dq_k| <= (|q_k| 2 eps / r^2 + 2 eps / r) / s, here with a factor 4 of slack
    (eps = 2^-24)."""
    eps = 2.0 ** -24
    r, s = np.asarray(r)[:, None], np.minimum(np.asarray(s), 1.0)[:, None]
    return 4 * (np.abs(q64) * 2 * eps / r ** 2 + 2 * eps / r) / s + 1e-30


def normal2rotation_torch32(n):
    """The reference's own float32 torch code (pcd.py:12-37), on whatever device n is."""
    import torch
    n = torch.nn.functional.normalize(n)
    w0 = torch.tensor([[1, 0, 0]], device=n.device).expand(n.shape)
    R0 = w0 - torch.sum(w0 * n, -1, True) * n
    R0 *= torch.sign(R0[:, :1])
    R0 = torch.nn.functional.normalize(R0)
    R1 = torch.cross(n, R0, dim=-1)
    R1 *= torch.sign(R1[:, 1:2]) * torch.sign(n[:, 2:])
    R = torch.stack([R0, R1, n], -1)
    tr = R[:, 0, 0] + R[:, 1, 1] + R[:, 2, 2] + 1e-6
    r = torch.sqrt(1 + tr) / 2
    return torch.stack([r, (R[:, 2, 1] - R[:, 1, 2]) / (4 * r), (R[:, 0, 2] - R[:, 2, 0]) / (4 * r),
                        (R[:, 1, 0] - R[:, 0, 1]) / (4 * r)], -1)


def sugar64(verts, faces, vnormals, colors, n):
    """mesh.py:212-250 per face and slot in float64 -> dict of xyz, normal (normalised), rgb, scale_xy, min_edge."""
    v, vn = np.asarray(verts, np.float64), np.asarray(vnormals, np.float64)
    B = np.asarray(np.float32(BARY[n]), np.float64)
    out = {k: [] for k in ("xyz", "normal", "rgb", "scale_xy", "min_edge")}
    for f in np.asarray(faces):
        p = v[f]
        m = min(np.linalg.norm(p[j] - p[(j + 1) % 3]) for j in range(3))
        for b in B:
            out["xyz"].append(b @ p)
            nr = b @ vn[f]
            out["normal"].append(nr / max(np.linalg.norm(nr), 1e-12))
            out["rgb"].append(b @ np.asarray(colors, np.float64)[f] if colors is not None else np.ones(3))
            out["min_edge"].append(m)
            out["scale_xy"].append(np.log(2 * max(m * RADIUS[n], 0.0) + 1e-7))
    return {k: np.array(x) for k, x in out.items()}


def dist2_64(xyz):
    """cKDTree(k=4) restated: mean over the 3 nearest other points of the squared distance (inf when missing)."""
    from scipy.spatial import cKDTree
    x = np.asarray(xyz, np.float64)
    k = min(4, len(x))
    d, _ = cKDTree(x).query(x, k=k)
    d = np.asarray(d).reshape(len(x), k)[:, 1:] ** 2
    if k < 4:
        d = np.concatenate([d, np.full((len(x), 4 - k), np.inf)], 1)
    return d.mean(1)
