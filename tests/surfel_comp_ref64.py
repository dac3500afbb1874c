"""Float64 reference of the surfel compositing: the 18 per-Gaussian sums k_surfel_render_bwd adds to the accumulator,
and the forward's per-pixel maps, each with a magnitude that bounds what float32 arithmetic can do to it.

Inputs are the forward's own per-Gaussian records (mean2D, Tu, Tv, Tw, opacity, the float32 view depth that is the sort
key, n_view, rgb) and the integer radii, promoted to float64, so that the projection's rounding does not enter.  Per-tile
lists are built here: the kernel's tile_rect in float32 on the record's mean2D and the integer radius (every tile of
the rect, no exact tile culling), sorted by (float32 depth, index).  The GPU's binned list is not used.

A pixel (x, y) (integer coordinates) walks its tile's list front to back with the contract's rules (DESIGN.md §3, surfel
rasterizer): k = x Tw - Tu, l = y Tw - Tv, p = k x l; the pair is skipped when p.z == 0; s = p.xy / p.z,
rho3 = |s|^2, rho2 = 2 |mean2D - (x, y)|^2, z = s.Tw.xy + Tw.z if rho3 <= rho2 else Tw.z, skipped when z < 0.2;
alpha = min(0.99, o G), G = exp(-min(rho3, rho2) / 2), skipped when alpha < 1/255; the pixel ends before a pair with
T (1 - alpha) < 1e-4; the median splat is the last one blended while T > 0.5.

Closed forms (written from the math, not from the kernel).  Transmittances are forward products T_i = prod_{k<i}
(1 - alpha_k), w_i = alpha_i T_i.  With s_j = gC.rgb_j + gD z_j + gN.n_j + gDist e_j the blended quantities against
their upstream,
    dL/dalpha_i = s_i T_i - (sum_{j behind i} s_j w_j + T_f (gC.bg - gA)) / (1 - alpha_i)
(gA: the upstream of the 1 - T channel).  The distortion dist = sum_{i<j} w_i w_j (m_i - m_j)^2 has
    d dist / d w_j = e_j = m_j^2 (1 - T_f) - 2 m_j M1 + M2,   d dist / d m_j = 2 w_j (m_j (1 - T_f) - M1)
with M1 = sum w m, M2 = sum w m^2 the pixel's final sums and m = 100/99.8 (1 - 0.2/z).  dL/dz_i = gD w_i +
gDist 2 w_i (m_i (1 - T_f) - M1) m'(z_i) + gMed [i is the median].  The 0.99 clamp passes no alpha gradient (it does
pass the z gradient).  The chain to the record fields: alpha = o G, rho = rho3 (ray-splat branch: s = p.xy / p.z,
p = k x l, k = x Tw - Tu, l = y Tw - Tv, and z through s and Tw) or rho2 (low-pass branch: mean2D, and z = Tw.z).

Output layout per Gaussian (the kernel's): {mean2D x, y; Tu 3; Tv 3; Tw 3; n_view 3; opacity; rgb 3}, `NAMES`.

Error model.  u = 2^-24.  Every quantity x of a pair is bounded by a magnitude xbar >= |x| with a float32 error
<= c u xbar:
  * k = x Tw - Tu, l = y Tw - Tv: each component one FFMA on exact inputs (the record fields and the integer pixel
    coordinate), so |dk| <= u |k| and |dl| <= u |l|.  nvcc contracts them so at -O3 with the default -fmad=true;
    `test_ray_splat_rows_are_single_ffmas` (tests/test_surfel_comp_ref64.py) pins that in the SASS of both
    compositing kernels, since a separate multiply and subtract would cost u |x Tw| (~1000 |k| at 1080p);
  * p = k x l: each component one FMUL and one FFMA: |dp| <= 4 u pbar, pbar = |k| x |l| with every product taken
    positive (2 u from the errors of k and l, 2 u from the two roundings); kappa = pbar.z / |p.z| is the condition
    number of the division by p.z;
  * s = p.xy / p.z (IEEE division): |ds| <= 5 u sigma, sigma = (pbar.xy + |s| pbar.z) / |p.z| >= |s|;
  * rho3: |d rho3| <= 10 u |s|.sigma + 2 u rho3 <= 12 u |s|.sigma; rho2 (mean2D - x rounded once): <= 4 u rho2;
  * G = expf(-rho/2) (precise expf: 2 ulp, argument rounding u rho/2) and alpha = o G: relative error u g_alpha,
    g_alpha = 3 + rho/2 + 6 |s|.sigma (ray-splat branch) or 3 + 2.5 rho2 (low-pass branch);
  * z: |dz| <= 5 u zbar, zbar = |Tw.x| sigma.x + |Tw.y| sigma.y + |Tw.z| (Tw.z exactly in the low-pass branch); m and
    m' = dm/dz carry 5 m' zbar + 5 (absolute, the 0.2f and 100/99.8 constants included) and 14 zbar / z + 4 (relative);
  * T: the forward multiplies (1 - alpha_k) front to back and stores T_f; the backward recovers T_i by IEEE division
    T / (1 - alpha_k) back to front.  Each factor costs <= u (2 + alpha_k g_k) / (1 - alpha_k) and T_i collects the
    forward's factors and the backward's: relative error <= 2 u K, K = sum over the pixel's contributors of
    (2 + alpha_k g_k) / (1 - alpha_k).  K >= 2 n also covers the n-step "behind" recursions of the backward (3 u per
    step on a convex combination) and the forward's running sums (C, D, N, M1, M2, dist);
  * the pair's terms couple to every contributor of the pixel (through T, the behind sums and M1 / M2): their alpha
    errors enter with the pixel's largest g_alpha, gpix, counted twice (alpha in w and G in the opacity chain);
  * float32 sums of the pairs: the 32-lane shuffle butterfly (5 levels) and one red.global per (warp, Gaussian):
    <= (5 + n_red) u times the sum of absolute values, n_red the number of warps, over every tile, in which the
    Gaussian has a contributor (an upper bound of its red.global count).
  The magnitude A of a sum is the same sum over the pairs with every signed factor replaced by its bar (the distortion's
  e by m^2 (1 - T_f) + 2 m M1 + M2), each pair weighted by its gain
    Gamma = 2 gpix + 4 K + 4 kappa + 14 zbar / z + 70 + 5 + n_red
  (15 for the three uses of s, 5 for z, 7 for m, the rest for the ~40 rounding steps of a pair's chain).  That is a
  first-order bound of the float32 error in units of u; EPS = 2 u leaves a factor two for the second-order terms.
  The forward maps use the same bars with Gamma_f = gpix + 2 K + 30 (no chain, no reduction).

Ambiguity.  A pixel is flagged when one of its decisions lies within FLAG_TOL times the first-order error of that
decision (from the records, not from the inputs): alpha vs 1/255 and o G vs 0.99 (relative u g_alpha), T (1 - alpha)
vs 1e-4 (relative u (g_alpha + 2 K)), rho3 vs rho2 (u (12 |s|.sigma + 4 rho2)), z vs 0.2 (u (5 zbar + 1)), p.z vs 0
(4 u pbar.z).  Only decisions the walk takes count: pairs up to and including the one that ends the pixel.
`flag`: zero upstream on every channel; `flag_median` (T vs 0.5 at a contributor, relative u (2 K + gpix)): only the
median-depth upstream is zeroed, since that decision moves nothing but the median gradient.  `masked(img, amap)`
applies both, and `sums` applies it by default.
"""
import numpy as np
import torch

F64 = torch.float64
TILE = 16
ALPHA_MIN = 1.0 / 255.0
ALPHA_MAX = 0.99
T_MIN = 1e-4
NEAR, FAR = 0.2, 100.0
MC = FAR / (FAR - NEAR)
U = 2.0 ** -24
EPS = 2 * U
FLAG_TOL = 2.0  # in units of the decision's first-order float32 error (the factor 2 of EPS)
NAMES = ("mean2D.x", "mean2D.y", "Tu.x", "Tu.y", "Tu.z", "Tv.x", "Tv.y", "Tv.z", "Tw.x", "Tw.y", "Tw.z",
         "n.x", "n.y", "n.z", "opacity", "r", "g", "b")
MAP_NAMES = ("D", "1-T", "n.x", "n.y", "n.z", "median depth", "distortion")


def _t64(x):
    if torch.is_tensor(x):
        return x.detach().to("cpu", F64)
    return torch.as_tensor(np.asarray(x), dtype=F64)


def unpack_records(recA, recB):
    """The kernel's two record arrays (recA [P,3] float4 = [P,12] floats, recB [P,2] float4 = [P,8]) -> dict of
    float32 tensors: mean2D [P,2], Tu, Tv, Tw, nv, rgb [P,3], opacity, depth [P]."""
    A = torch.as_tensor(recA).reshape(-1, 12).float().cpu()
    B = torch.as_tensor(recB).reshape(-1, 8).float().cpu()
    return dict(mean2D=A[:, 0:2], Tw=A[:, 2:5], opacity=A[:, 5], depth=A[:, 6], Tu=A[:, 8:11],
                Tv=torch.stack([A[:, 11], B[:, 0], B[:, 1]], 1), nv=B[:, 2:5], rgb=B[:, 5:8])


def surfel_rects(mean2D, radii, W, H):
    """The kernel's tile_rect in float32: x0 = (px - r) / 16, x1 = (px + r + 16 - 1) / 16 (left to right),
    truncated toward zero and clamped to the grid -> int64 [P,4] (x0, y0, x1, y1) and the grid size."""
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    m = np.asarray(torch.as_tensor(mean2D).detach().cpu().numpy(), dtype=np.float32).reshape(-1, 2)
    r = np.asarray(torch.as_tensor(radii).detach().cpu().numpy()).astype(np.int64).reshape(-1)
    rr, t, one = r.astype(np.float32), np.float32(TILE), np.float32(1)
    lo = lambda c: np.trunc((m[:, c] - rr) / t)
    hi = lambda c: np.trunc((((m[:, c] + rr) + t) - one) / t)
    x0, x1 = np.clip(lo(0), 0, gx).astype(np.int64), np.clip(hi(0), 0, gx).astype(np.int64)
    y0, y1 = np.clip(lo(1), 0, gy).astype(np.int64), np.clip(hi(1), 0, gy).astype(np.int64)
    return np.stack([x0, y0, x1, y1], 1), gx, gy


def tile_lists(mean2D, radii, depth, W, H, tiles=None):
    """Per-tile Gaussian lists: every tile of each live Gaussian's rect, sorted by (float32 depth, index)."""
    rc, gx, gy = surfel_rects(mean2D, radii, W, H)
    r = np.asarray(torch.as_tensor(radii).cpu().numpy()).reshape(-1)
    key = np.asarray(torch.as_tensor(depth).cpu().numpy(), dtype=np.float32).reshape(-1)
    order = np.lexsort((np.arange(len(key)), key))
    want = None if tiles is None else set(int(t) for t in tiles)
    lists = [[] for _ in range(gx * gy)]
    for i in order:
        x0, y0, x1, y1 = rc[i]
        if r[i] <= 0 or (x1 - x0) * (y1 - y0) == 0:
            continue
        for ty in range(y0, y1):
            for tx in range(x0, x1):
                t = ty * gx + tx
                if want is None or t in want:
                    lists[t].append(int(i))
    return lists, gx, gy


def _cross(a, b):
    return torch.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                        a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def _cross_abs(a, b):
    """|a| x |b| with every product taken positive (the magnitude of a cross product's terms)."""
    a, b = a.abs(), b.abs()
    return torch.stack([a[..., 1] * b[..., 2] + a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] + a[..., 0] * b[..., 2],
                        a[..., 0] * b[..., 1] + a[..., 1] * b[..., 0]], -1)


def m_of(z):
    return MC * (1 - NEAR / z)


def dm_of(z):
    return MC * NEAR / (z * z)


class SurfelCompositing:
    """The geometry half of the reference for one forward: per-tile lists, the walk of every pixel, flags and gains.
    `sums(img, amap)` then gives the 18 sums for any upstream; `maps()` the forward's per-pixel maps.
    tiles: build only these tiles (the upstream must be confined to them)."""

    def __init__(self, rec, radii, W, H, bg, tiles=None, dtype=F64):
        self.W, self.H, self.dt = int(W), int(H), dtype
        cv = lambda x: _t64(x).to(dtype)
        self.m2, self.Tu, self.Tv, self.Tw = cv(rec["mean2D"]), cv(rec["Tu"]), cv(rec["Tv"]), cv(rec["Tw"])
        self.nv, self.rgb, self.o = cv(rec["nv"]), cv(rec["rgb"]), cv(rec["opacity"]).reshape(-1)
        self.bg = cv(bg).reshape(3)
        self.P = self.m2.shape[0]
        lists, self.gx, self.gy = tile_lists(rec["mean2D"], radii, rec["depth"], W, H, tiles)
        HW = self.W * self.H
        self.flag = torch.zeros(HW, dtype=torch.bool)
        self.flag_median = torch.zeros(HW, dtype=torch.bool)
        self.flag_kinds = {k: torch.zeros(HW, dtype=torch.bool) for k in
                           ("alpha", "clamp", "stop", "branch", "near", "pz", "median")}
        self.built = torch.zeros(HW, dtype=torch.bool)    # pixels of the tiles built
        self.covered = torch.zeros(HW, dtype=torch.bool)  # at least one contributor
        self.n_contrib = torch.zeros(HW, dtype=torch.int64)
        self.last = torch.zeros(HW, dtype=torch.int64)    # 1 + list position of the last contributor (n_contrib)
        self.ended = torch.zeros(HW, dtype=torch.bool)
        self.median = torch.full((HW,), -1, dtype=torch.int64)
        self.clamped_pairs = 0
        self.n_red = torch.zeros(self.P, dtype=dtype)  # warps, over every tile, in which a Gaussian has a contributor
        self.tiles = []
        want = None if tiles is None else set(int(v) for v in tiles)
        for t, ids in enumerate(lists):
            if ids:
                self.tiles.append(self._tile(t, torch.as_tensor(ids)))
            elif want is None or t in want:
                self._mark_built(t)

    def _pixels(self, t):
        tx, ty = t % self.gx, t // self.gx
        k = torch.arange(TILE * TILE)
        px, py = tx * TILE + k % TILE, ty * TILE + k // TILE
        inside = (px < self.W) & (py < self.H)
        return px[inside], py[inside], k[inside]

    def _mark_built(self, t):
        px, py, _ = self._pixels(t)
        self.built[py * self.W + px] = True

    def _tile(self, t, ids):
        dt = self.dt
        px, py, lane = self._pixels(t)
        pid = py * self.W + px
        self.built[pid] = True
        Np, n = pid.numel(), ids.numel()
        x = px.to(dt)[:, None, None]
        y = py.to(dt)[:, None, None]
        Tu, Tv, Tw = self.Tu[ids][None], self.Tv[ids][None], self.Tw[ids][None]
        # the kernel's single FFMAs (exact product, one rounding); in float64 the product and difference are exact enough
        k = (x.double() * Tw.double() - Tu.double()).to(dt)
        l = (y.double() * Tw.double() - Tv.double()).to(dt)
        kbar, lbar = k.abs(), l.abs()  # single FFMAs on exact inputs: |dk| <= u |k|
        p = _cross(k, l)
        pbar = _cross_abs(k, l)
        pz_ok = p[..., 2] != 0
        pz = torch.where(pz_ok, p[..., 2], torch.ones_like(p[..., 2]))
        sx, sy = p[..., 0] / pz, p[..., 1] / pz
        apz = pz.abs()
        kappa = pbar[..., 2] / apz
        sigx = (pbar[..., 0] + sx.abs() * pbar[..., 2]) / apz
        sigy = (pbar[..., 1] + sy.abs() * pbar[..., 2]) / apz
        rho3 = sx * sx + sy * sy
        dx = self.m2[ids, 0][None] - x[..., 0]
        dy = self.m2[ids, 1][None] - y[..., 0]
        rho2 = 2 * (dx * dx + dy * dy)
        use3 = rho3 <= rho2
        rho = torch.where(use3, rho3, rho2)
        Twx, Twy, Twz = Tw[..., 0], Tw[..., 1], Tw[..., 2]
        z = torch.where(use3, sx * Twx + sy * Twy + Twz, Twz.expand_as(sx))
        zbar = torch.where(use3, Twx.abs() * sigx + Twy.abs() * sigy + Twz.abs(), Twz.abs().expand_as(sx))
        zok = pz_ok & (z >= NEAR)
        G = torch.exp(-0.5 * rho)
        o = self.o[ids][None]
        oG = o * G
        alpha = oG.clamp(max=ALPHA_MAX)
        valid = zok & (alpha >= ALPHA_MIN)
        ssig = sx.abs() * sigx + sy.abs() * sigy
        g_alpha = torch.where(use3, 3 + rho / 2 + 6 * ssig, 3 + 2.5 * rho2)
        av = torch.where(valid, alpha, torch.zeros_like(alpha))
        incl = torch.cumprod(1 - av, dim=1)
        pos = torch.arange(n)[None, :]
        ends = valid & (incl < T_MIN)
        kstop = torch.where(ends.any(1), ends.to(torch.int8).argmax(1), torch.full((Np,), n))
        contrib = valid & (pos < kstop[:, None])
        a = torch.where(contrib, alpha, torch.zeros_like(alpha))
        T = torch.cumprod(torch.cat([torch.ones(Np, 1, dtype=dt), 1 - a], 1), dim=1)
        T_f, T = T[:, -1], T[:, :-1]
        w = a * T
        medm = contrib & (T > 0.5)
        med_pos = (medm.long() * (pos + 1)).max(1).values - 1  # -1: none
        med = torch.zeros_like(contrib)
        has_med = med_pos >= 0
        med[has_med.nonzero().flatten(), med_pos[has_med]] = True
        zs = torch.where(contrib, z, torch.ones_like(z))
        m, dm = m_of(zs), dm_of(zs)
        mbar = m.abs() + dm * zbar + 1  # |m| <= 1.002; the +1 carries the absolute rounding of 1 - 0.2/z
        gpix = torch.where(contrib, g_alpha, torch.zeros_like(g_alpha)).max(1).values
        K = torch.where(contrib, (2 + a * g_alpha) / (1 - a), torch.zeros_like(a)).sum(1)

        # ambiguity flags, on decisions the walk takes
        reach = pos <= kstop[:, None]
        tol = FLAG_TOL * U
        # relative distance to a threshold, as |log(v / thr)| (G's relative error is the absolute error of log G)
        near_rel = lambda v, thr, rel: torch.log(v.clamp(min=1e-300) / thr).abs() <= tol * rel
        vis = reach & pz_ok & (o * torch.exp(-0.5 * torch.minimum(rho3, rho2)) >= 0.5 * ALPHA_MIN)
        f_pz = (reach & (o >= ALPHA_MIN) & (p[..., 2].abs() <= tol * 4 * pbar[..., 2])).any(1)
        f_branch = (vis & ((rho3 - rho2).abs() <= tol * (12 * ssig + 4 * rho2))).any(1)
        f_near = (vis & ((z - NEAR).abs() <= tol * (5 * zbar + 1))).any(1)
        f_alpha = (reach & zok & near_rel(oG, ALPHA_MIN, g_alpha)).any(1)
        f_clamp = (reach & zok & near_rel(oG, ALPHA_MAX, g_alpha)).any(1)
        f_stop = (reach & valid & near_rel(incl, T_MIN, g_alpha + 2 * K[:, None])).any(1)
        f_med = (contrib & near_rel(T, 0.5, gpix[:, None] + 2 * K[:, None])).any(1)
        for name, f in (("alpha", f_alpha), ("clamp", f_clamp), ("stop", f_stop), ("branch", f_branch),
                        ("near", f_near), ("pz", f_pz), ("median", f_med)):
            self.flag_kinds[name][pid] = f
        self.flag[pid] = f_alpha | f_clamp | f_stop | f_branch | f_near | f_pz
        self.flag_median[pid] = f_med
        self.covered[pid] = contrib.any(1)
        self.n_contrib[pid] = contrib.sum(1)
        self.last[pid] = (contrib.long() * (pos + 1)).max(1).values
        self.ended[pid] = kstop < n
        self.median[pid[has_med]] = ids[med_pos[has_med]]
        self.clamped_pairs += int((contrib & (oG > ALPHA_MAX)).sum())
        # warps (two rows of 16 pixels) in which the Gaussian has a contributor: its red.global count from this tile
        warp = lane // 32
        n_warp = torch.zeros(n, dtype=dt)
        for wv in torch.unique(warp).tolist():
            n_warp += contrib[warp == wv].any(0).to(dt)
        self.n_red.index_add_(0, ids, n_warp)
        return dict(ids=ids, pid=pid, x=x[..., 0], y=y[..., 0], k=k, l=l, kbar=kbar, lbar=lbar, sx=sx, sy=sy,
                    sigx=sigx, sigy=sigy, apz=apz, pz=pz, kappa=kappa, dx=dx, dy=dy, use3=use3, z=z, zbar=zbar,
                    G=G, o=o, oG=oG, a=a, T=T, T_f=T_f, w=w, med=med, m=m, dm=dm, mbar=mbar, gpix=gpix, K=K,
                    contrib=contrib, Twx=Twx, Twy=Twy)

    # ---- upstream --------------------------------------------------------------------------------------------------
    def masked(self, img, amap):
        """img [3,H,W], amap [9,H,W] (torch) with the flagged pixels zeroed (only the median-depth channel at
        flag_median pixels)."""
        keep = (~self.flag).reshape(self.H, self.W)
        keep_m = keep & (~self.flag_median).reshape(self.H, self.W)
        img = torch.where(keep, img, torch.zeros((), dtype=img.dtype))
        amap = torch.where(keep, amap, torch.zeros((), dtype=amap.dtype)).clone()
        amap[5] = torch.where(keep_m, amap[5], torch.zeros((), dtype=amap.dtype))
        return img, amap

    def sums(self, img, amap, drop_flagged=True):
        """-> (S [P,18], A [P,18]) for the upstream img [3,H,W] and amap [9,H,W] (channels 7-8 carry no gradient).
        Also sets self.reached: the Gaussians that contribute to a pixel with non-zero upstream on channels 0-6."""
        dt = self.dt
        if drop_flagged:
            img, amap = self.masked(img, amap)
        HW = self.W * self.H
        gi = _t64(img).to(dt).reshape(3, HW)
        gm = _t64(amap).to(dt).reshape(9, HW)
        nz = (gi != 0).any(0) | (gm[:7] != 0).any(0)
        S = torch.zeros(self.P, 18, dtype=dt)
        Aall = torch.zeros(self.P, 18, dtype=dt)
        self.reached = torch.zeros(self.P, dtype=torch.bool)
        for tl in self.tiles:
            ids, pid = tl["ids"], tl["pid"]
            col = lambda v: v[:, None]
            gC = [col(gi[c, pid]) for c in range(3)]
            gN = [col(gm[2 + c, pid]) for c in range(3)]
            gD, gA, gMed, gDist = col(gm[0, pid]), col(gm[1, pid]), col(gm[5, pid]), col(gm[6, pid])
            rgb = [self.rgb[ids, c][None] for c in range(3)]
            nv = [self.nv[ids, c][None] for c in range(3)]
            ct, w, T, T_f, a = tl["contrib"], tl["w"], tl["T"], tl["T_f"], tl["a"]
            z, zbar, m, dm, mbar = tl["z"], tl["zbar"], tl["m"], tl["dm"], tl["mbar"]
            Af = col(1 - T_f)
            M1, M2 = col((w * m).sum(1)), col((w * m * m).sum(1))
            M1b, M2b = col((w * mbar).sum(1)), col((w * mbar * mbar).sum(1))
            e = m * m * Af - 2 * m * M1 + M2
            ebar = mbar * mbar * Af + 2 * mbar * M1b + M2b
            s = sum(gC[c] * rgb[c] + gN[c] * nv[c] for c in range(3)) + gD * z + gDist * e
            sbar = sum(gC[c].abs() * rgb[c].abs() + gN[c].abs() * nv[c].abs() for c in range(3)) + \
                gD.abs() * zbar + gDist.abs() * ebar
            bgd = sum(gC[c][:, 0] * self.bg[c] for c in range(3)) - gA[:, 0]
            bgb = sum(gC[c][:, 0].abs() * self.bg[c].abs() for c in range(3)) + gA[:, 0].abs()
            sw, swb = s * w, sbar * w
            inv1a = 1 / (1 - a)
            behind = sw.flip(1).cumsum(1).flip(1) - sw + col(T_f * bgd)
            behindb = swb.flip(1).cumsum(1).flip(1) - swb + col(T_f * bgb)
            dal = torch.where(ct, s * T - behind * inv1a, torch.zeros_like(w))
            dalb = torch.where(ct, sbar * T + behindb * inv1a, torch.zeros_like(w))
            medf = tl["med"].to(dt)
            gz = gD * w + gDist * 2 * w * (m * Af - M1) * dm + gMed * medf
            gzb = gD.abs() * w + gDist.abs() * 2 * w * (mbar * Af + M1b) * dm + gMed.abs() * medf
            G, o = tl["G"], tl["o"]
            unclamped = (tl["oG"] <= ALPHA_MAX) & ct
            zero = torch.zeros_like(w)
            acc_o = torch.where(unclamped, dal * G, zero)
            acc_ob = torch.where(unclamped, dalb * G, zero)
            drho = torch.where(unclamped, -0.5 * G * o * dal, zero)
            drhob = torch.where(unclamped, 0.5 * G * o * dalb, zero)
            u3 = tl["use3"] & ct
            u2 = ~tl["use3"] & ct
            sx, sy, sigx, sigy, pz, apz = tl["sx"], tl["sy"], tl["sigx"], tl["sigy"], tl["pz"], tl["apz"]
            Twx, Twy = tl["Twx"], tl["Twy"]
            gsx = drho * 2 * sx + gz * Twx
            gsy = drho * 2 * sy + gz * Twy
            gsxb = drhob * 2 * sigx + gzb * Twx.abs()
            gsyb = drhob * 2 * sigy + gzb * Twy.abs()
            gp = torch.stack([gsx / pz, gsy / pz, -(gsx * sx + gsy * sy) / pz], -1)
            gpb = torch.stack([gsxb / apz, gsyb / apz, (gsxb * sigx + gsyb * sigy) / apz], -1)
            gk, gl = _cross(tl["l"], gp), _cross(gp, tl["k"])
            gkb, glb = _cross_abs(tl["lbar"], gpb), _cross_abs(gpb, tl["kbar"])
            xx, yy = tl["x"], tl["y"]
            sel3 = lambda v: torch.where(u3, v, zero)
            sel2 = lambda v: torch.where(u2, v, zero)
            terms = [sel2(drho * 4 * tl["dx"]), sel2(drho * 4 * tl["dy"])]
            bars = [sel2(drhob * 4 * tl["dx"].abs()), sel2(drhob * 4 * tl["dy"].abs())]
            terms += [sel3(-gk[..., c]) for c in range(3)] + [sel3(-gl[..., c]) for c in range(3)]
            bars += [sel3(gkb[..., c]) for c in range(3)] + [sel3(glb[..., c]) for c in range(3)]
            terms += [sel3(gz * sx + xx * gk[..., 0] + yy * gl[..., 0]), sel3(gz * sy + xx * gk[..., 1] + yy * gl[..., 1]),
                      sel3(gz + xx * gk[..., 2] + yy * gl[..., 2]) + sel2(gz)]
            bars += [sel3(gzb * sigx + xx.abs() * gkb[..., 0] + yy.abs() * glb[..., 0]),
                     sel3(gzb * sigy + xx.abs() * gkb[..., 1] + yy.abs() * glb[..., 1]),
                     sel3(gzb + xx.abs() * gkb[..., 2] + yy.abs() * glb[..., 2]) + sel2(gzb)]
            terms += [w * gN[c] for c in range(3)] + [acc_o] + [w * gC[c] for c in range(3)]
            bars += [w * gN[c].abs() for c in range(3)] + [acc_ob] + [w * gC[c].abs() for c in range(3)]
            zr = torch.where(u3, zbar / z.abs().clamp(min=NEAR), zero)
            gain = 2 * col(tl["gpix"]) + 4 * col(tl["K"]) + 4 * torch.where(u3, tl["kappa"], zero) + 14 * zr + 75 + \
                self.n_red[ids][None]
            self.reached[ids[(ct & col(nz[pid])).any(0)]] = True
            S.index_add_(0, ids, torch.stack([v.sum(0) for v in terms], 1))
            Aall.index_add_(0, ids, torch.stack([(b * gain).sum(0) for b in bars], 1))
        return S, Aall

    # ---- forward ---------------------------------------------------------------------------------------------------
    def maps(self):
        """The forward's per-pixel values from the same walk -> dict name -> (value [..., HW], magnitude); image [3,HW],
        D, 1-T, normal [3,HW], median depth, distortion, and the median id [HW] (-1: none; no magnitude)."""
        dt, HW = self.dt, self.W * self.H
        img = self.bg[:, None].repeat(1, HW)  # pixels no splat reaches show the background
        imgA = self.bg.abs()[:, None].repeat(1, HW)
        out = {k: (torch.zeros(HW, dtype=dt), torch.zeros(HW, dtype=dt)) for k in ("D", "1-T", "median depth",
                                                                                    "distortion")}
        nrm, nrmA = torch.zeros(3, HW, dtype=dt), torch.zeros(3, HW, dtype=dt)
        Tall = torch.ones(HW, dtype=dt)
        for tl in self.tiles:
            ids, pid, w, T, T_f, ct = tl["ids"], tl["pid"], tl["w"], tl["T"], tl["T_f"], tl["contrib"]
            gam = tl["gpix"] + 2 * tl["K"] + 30
            Tall[pid] = T_f
            for c in range(3):
                img[c, pid] = (w * self.rgb[ids, c][None]).sum(1) + T_f * self.bg[c]
                imgA[c, pid] = ((w * self.rgb[ids, c][None].abs()).sum(1) + T_f * self.bg[c].abs()) * gam
                nrm[c, pid] = (w * self.nv[ids, c][None]).sum(1)
                nrmA[c, pid] = (w * self.nv[ids, c][None].abs()).sum(1) * gam
            out["D"][0][pid] = (w * tl["z"]).sum(1)
            out["D"][1][pid] = (w * tl["zbar"]).sum(1) * gam
            out["1-T"][0][pid] = 1 - T_f
            out["1-T"][1][pid] = gam
            md = tl["med"]
            out["median depth"][0][pid] = torch.where(md, tl["z"], torch.zeros_like(w)).sum(1)
            out["median depth"][1][pid] = torch.where(md, tl["zbar"], torch.zeros_like(w)).sum(1) * gam
            # running sums in front of each splat, as the forward accumulates them
            m, mb = tl["m"], tl["mbar"]
            M1 = (w * m).cumsum(1) - w * m
            M2 = (w * m * m).cumsum(1) - w * m * m
            M1b = (w * mb).cumsum(1) - w * mb
            M2b = (w * mb * mb).cumsum(1) - w * mb * mb
            out["distortion"][0][pid] = (w * (m * m * (1 - T) + M2 - 2 * m * M1)).sum(1)
            out["distortion"][1][pid] = (w * (mb * mb * (1 - T) + M2b + 2 * mb * M1b)).sum(1) * gam
        out["image"] = (img, imgA)
        out["normal"] = (nrm, nrmA)
        out["final T"] = Tall
        out["median id"] = self.median.clone()
        return out

    def stats(self):
        cov = int(self.covered.sum())
        return dict(covered=cov, flagged=int((self.flag & self.covered).sum()),
                    frac=float((self.flag & self.covered).sum()) / max(cov, 1),
                    median_frac=float((self.flag_median & self.covered).sum()) / max(cov, 1),
                    kinds={k: int((v & self.covered).sum()) for k, v in self.flag_kinds.items()})


def worst_ratio(got, ref, Am, eps=EPS):
    """max over every element of |got - ref| / (eps A) -> (ratio, row, column); exact agreement counts 0."""
    got, ref, Am = _t64(got), _t64(ref), _t64(Am)
    if got.dim() == 1:
        got, ref, Am = got[:, None], ref[:, None], Am[:, None]
    if not torch.isfinite(got).all():
        i = int((~torch.isfinite(got)).nonzero()[0, 0])
        return float("inf"), i, -1
    e = (got - ref).abs()
    r = torch.where(e == 0, torch.zeros_like(e), e / (eps * Am + 1e-300))
    flat = int(r.argmax())
    return float(r.reshape(-1)[flat]), flat // r.shape[1], flat % r.shape[1]
