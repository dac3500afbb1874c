"""Float64 restatement of the Shape-as-Points meshing (DESIGN.md 7h; the reference's models/sap.py and the DPSR of
utils/graphics_utils.py with res = 256, sig = 2, scale = shift = True, weighted = False), with numpy's FFT:

  normalize64(xyz)                 c = mean, s = 1.2 max|xyz - c|, p = ((xyz - c)/s + 1)/2
  splat64(p, normals, res)         point_rasterize(weighted=False): trilinear, node i0 + 1 wrapped to 0 at res
  dpsr64(p, normals, res, sig)     the spectral solve, shift and scale -> dict(grid, phi, off, fv0, psi)
  marching_cubes64(psi)            marching cubes at 0 with the project's tables, faces facing psi > 0; index coordinates
  mesh64(xyz, normals, res, sig)   the whole chain, vertices in world coordinates

Plus the checkers the tests share (trilinear interpolation, edge-manifold statistics, Chamfer distance).
"""
import numpy as np

from oracle.tsdf_oracle import MC_EDGE, MC_NTRI, MC_TRI

U32 = 2.0 ** -24  # unit roundoff of float32


def normalize64(xyz):
    xyz = np.asarray(xyz, np.float64)
    c = xyz.mean(0)
    s = 1.2 * np.abs(xyz - c).max()
    return ((xyz - c) / s + 1.0) / 2.0, c, s


def axis_weights(p, res):
    """-> (i0 [N,3] int, w [2,N,3]): weight w[0] towards node i0, w[1] towards node (i0 + 1) mod res, per axis."""
    t = np.asarray(p, np.float64) * res
    i0 = np.floor(t)
    return i0.astype(np.int64), np.stack([i0 + 1.0 - t, t - i0])


def corners():
    """The 8 offsets o = (ox, oy, oz) in x-major order (the reference's meshgrid order)."""
    return [((o >> 2) & 1, (o >> 1) & 1, o & 1) for o in range(8)]


def splat64(p, normals, res):
    """-> grid [3,res,res,res] float64 and the per-node sum of |terms| (for rounding bounds)."""
    i0, w = axis_weights(p, res)
    n = np.asarray(normals, np.float64)
    grid = np.zeros((3, res ** 3))
    mag = np.zeros(res ** 3)
    for ox, oy, oz in corners():
        wt = w[ox, :, 0] * w[oy, :, 1] * w[oz, :, 2]
        node = (((i0[:, 0] + ox) % res) * res + (i0[:, 1] + oy) % res) * res + (i0[:, 2] + oz) % res
        for d in range(3):
            np.add.at(grid[d], node, wt * n[:, d])
        np.add.at(mag, node, wt * np.abs(n).max(1))
    return grid.reshape(3, res, res, res), mag.reshape(res, res, res)


def omega(res):
    """Integer frequencies [res,res,res//2+1,3]: fftfreq on the first two axes, rfftfreq on the last."""
    f = np.fft.fftfreq(res, d=1.0 / res)
    r = np.fft.rfftfreq(res, d=1.0 / res)
    return np.stack(np.meshgrid(f, f, r, indexing="ij"), -1)


def spectral64(grid, res, sig):
    """phi = irfftn(-i sum_d 2 pi w_d G N_d / (-sum_d (2 pi w_d)^2 + 1e-6)), 0 at w = 0."""
    spec = np.fft.rfftn(grid, axes=(1, 2, 3))
    om = omega(res)
    G = np.exp(-0.5 * (sig * 2.0 * np.sqrt((om ** 2).sum(-1)) / res) ** 2)
    w = 2.0 * np.pi * om
    div = -1j * sum(w[..., d] * G * spec[d] for d in range(3))
    phi_hat = div / (-(w ** 2).sum(-1) + 1e-6)
    phi_hat[0, 0, 0] = 0.0
    return np.fft.irfftn(phi_hat, s=(res, res, res), axes=(0, 1, 2))


def interp64(grid, p):
    """grid_interp: trilinear interpolation of grid [res,res,res] at p [N,3] (same weights as the splat)."""
    res = grid.shape[0]
    i0, w = axis_weights(p, res)
    out = np.zeros(len(i0))
    for ox, oy, oz in corners():
        out += grid[(i0[:, 0] + ox) % res, (i0[:, 1] + oy) % res, (i0[:, 2] + oz) % res] * \
            (w[ox, :, 0] * w[oy, :, 1] * w[oz, :, 2])
    return out


def dpsr64(p, normals, res, sig=2.0):
    grid, mag = splat64(p, normals, res)
    phi = spectral64(grid, res, sig)
    off = interp64(phi, p).mean()
    fv0 = phi[0, 0, 0] - off
    scaled = -(phi - off) / abs(fv0) * 0.5
    return dict(grid=grid, mag=mag, phi=phi, off=off, fv0=fv0, scaled=scaled, psi=np.tanh(scaled))


def psi_bound(ref, res):
    """Bound on |psi - psi64| for a float32 pipeline: the splat weights and products round by <= 8u per term, and the
    forward and inverse FFTs each by ~2u log2(res^3) of the field's magnitude, so phi carries
    d_phi = u (8 + 4 log2(res^3)) max|phi - off|.  offset and fv0 are differences of such values (<= 2 d_phi each);
    with a = -(phi - off) / (2 |fv0|) that gives |d a| <= d_phi / |fv0| (1.5 + 2 max|a|), and tanh is 1-Lipschitz."""
    d_phi = U32 * (8.0 + 4.0 * np.log2(float(res) ** 3)) * np.abs(ref["phi"] - ref["off"]).max()
    return d_phi / abs(ref["fv0"]) * (1.5 + 2.0 * np.abs(ref["scaled"]).max())


def marching_cubes64(psi):
    """-> (vertices [V,3] float64 in index coordinates, faces [F,3] int64) in the order gsr_sap_marching_cubes
    emits them: vertices by node (x-major) then axis, faces by cube then table entry."""
    psi = np.asarray(psi, np.float64)
    r = psi.shape[0]
    outside = psi >= 0.0
    emask = np.zeros((r, r, r), np.int64)
    for a in range(3):
        sl0 = [slice(None)] * 3; sl1 = [slice(None)] * 3
        sl0[a] = slice(0, r - 1); sl1[a] = slice(1, r)
        cross = np.zeros((r, r, r), bool)
        cross[tuple(sl0)] = outside[tuple(sl0)] != outside[tuple(sl1)]
        emask |= cross.astype(np.int64) << a
    flat_mask = emask.reshape(-1)
    cnt = (flat_mask & 1) + ((flat_mask >> 1) & 1) + ((flat_mask >> 2) & 1)
    vbase = np.concatenate([[0], np.cumsum(cnt)])
    verts = np.zeros((vbase[-1], 3))
    g = np.arange(r ** 3)
    xyz = np.stack([g // (r * r), (g // r) % r, g % r], 1).astype(np.float64)
    step = np.array([r * r, r, 1])
    for a in range(3):
        has = ((flat_mask >> a) & 1).astype(bool)
        below = flat_mask & ((1 << a) - 1)
        slot = vbase[:-1] + (below & 1) + ((below >> 1) & 1)
        f0 = psi.reshape(-1)[has]
        f1 = psi.reshape(-1)[g[has] + step[a]]
        pos = xyz[has].copy()
        pos[:, a] += f0 / (f0 - f1)
        verts[slot[has]] = pos
    c = r - 1
    case = np.zeros((c, c, c), np.int64)
    for k in range(8):
        case |= outside[(k & 1):(k & 1) + c, ((k >> 1) & 1):((k >> 1) & 1) + c, ((k >> 2) & 1):((k >> 2) & 1) + c] \
            .astype(np.int64) << k
    cube_g = ((np.arange(c)[:, None, None] * r + np.arange(c)[None, :, None]) * r + np.arange(c)[None, None, :])
    case, cube_g = case.reshape(-1), cube_g.reshape(-1)
    nt = MC_NTRI[case].astype(np.int64)
    fbase = np.concatenate([[0], np.cumsum(nt)])
    faces = np.zeros((fbase[-1], 3), np.int64)
    for t in range(5):
        sel = nt > t
        cs = case[sel]
        for j in range(3):
            e = MC_TRI[cs, 3 * t + j].astype(np.int64)
            c0, ax = MC_EDGE[e, 0], MC_EDGE[e, 2]
            go = cube_g[sel] + (c0 & 1) * step[0] + ((c0 >> 1) & 1) * step[1] + ((c0 >> 2) & 1) * step[2]
            below = flat_mask[go] & ((1 << ax) - 1)
            faces[fbase[:-1][sel] + t, j] = vbase[go] + (below & 1) + ((below >> 1) & 1)
    return verts, faces


def mesh64(xyz, normals, res, sig=2.0):
    """The whole chain in float64 -> (vertices [V,3] world, faces [F,3], dpsr64 dict, c, s)."""
    p, c, s = normalize64(xyz)
    ref = dpsr64(p, normals, res, sig)
    v, f = marching_cubes64(ref["psi"])
    return (v / res * 2.0 - 1.0) * s + c, f, ref, c, s


def trilinear(psi, q):
    """Trilinear interpolation of psi [r,r,r] at index coordinates q [N,3] inside the grid (no wrap)."""
    r = psi.shape[0]
    i0 = np.clip(np.floor(q).astype(np.int64), 0, r - 2)
    t = q - i0
    out = np.zeros(len(q))
    for ox, oy, oz in corners():
        w = (t[:, 0] if ox else 1 - t[:, 0]) * (t[:, 1] if oy else 1 - t[:, 1]) * (t[:, 2] if oz else 1 - t[:, 2])
        out += w * psi[i0[:, 0] + ox, i0[:, 1] + oy, i0[:, 2] + oz]
    return out


def edge_manifold(faces):
    """-> (every edge in exactly two faces, consistently oriented; Euler characteristic V - E + F over used vertices)."""
    f = np.asarray(faces, np.int64)
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    key = np.minimum(e[:, 0], e[:, 1]) * (f.max() + 1) + np.maximum(e[:, 0], e[:, 1])
    _, cnt = np.unique(key, return_counts=True)
    directed = e[:, 0] * (f.max() + 1) + e[:, 1]
    oriented = len(np.unique(directed)) == len(directed)
    return bool((cnt == 2).all() and oriented), len(np.unique(f)) - len(cnt) + len(f)


def chamfer(a, b):
    """Symmetric mean nearest-neighbour distance between point sets a and b."""
    from scipy.spatial import cKDTree
    return 0.5 * (cKDTree(b).query(a)[0].mean() + cKDTree(a).query(b)[0].mean())


def sphere(n, r=0.5, centre=(0.1, -0.2, 0.3), seed=0):
    g = np.random.default_rng(seed)
    d = g.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return (np.asarray(centre) + r * d).astype(np.float32), d.astype(np.float32)


def torus(n, R=0.6, r=0.25, seed=1):
    g = np.random.default_rng(seed)
    u, v = g.uniform(0, 2 * np.pi, n), g.uniform(0, 2 * np.pi, n)
    ring = np.stack([np.cos(u), np.sin(u), np.zeros(n)], 1)
    nrm = ring * np.cos(v)[:, None] + np.array([0.0, 0.0, 1.0]) * np.sin(v)[:, None]
    return (R * ring + r * nrm).astype(np.float32), nrm.astype(np.float32)


def plane(n, seed=2):
    g = np.random.default_rng(seed)
    xy = g.uniform(-0.5, 0.5, (n, 2))
    z = 0.05 * np.sin(3 * xy[:, 0])
    nrm = np.stack([-0.15 * np.cos(3 * xy[:, 0]), np.zeros(n), np.ones(n)], 1)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    return np.column_stack([xy, z]).astype(np.float32), nrm.astype(np.float32)


SHAPES = {"sphere": lambda: sphere(1500), "torus": lambda: torus(2000), "plane": lambda: plane(1000)}
