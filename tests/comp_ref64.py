"""Float64 reference of the compositing backward: the ten per-Gaussian sums k_render_bwd adds to the accumulator.

Written from the math of front-to-back alpha compositing with the reference rasterizer's conventions, in torch
float64 and vectorised over the pixels of a tile.  It shares neither the kernel's single "behind" recurrence Q nor the
oracle's per-channel recurrences: transmittances are forward products and dL/dalpha is the closed form
    dL/dalpha_i = s_i T_i - (sum_{j behind i} s_j w_j + T_final bg.g) / (1 - alpha_i),   w_j = alpha_j T_j,
with s_i = rgb_i.g + depth_i gD + gO the five blended channels against their upstream.

Inputs are the forward's per-Gaussian state (means2D, conic_opacity, rgb, depths, radii), promoted to float64, and
the four upstream images.  Per-tile lists are built here from the tile rectangles (the rasterizer's getRect on the
same float32 values) and sorted by (float32 depth, index); the GPU's binned list is not used.  A pixel walks its list
with the reference's thresholds: power > 0 and alpha < 1/255 skip a pair, alpha = min(0.99, o G), T (1 - alpha) <
1e-4 ends the pixel before that pair blends, and the median-depth Gaussian is the one at which T crosses 0.5.

Output layout per Gaussian (the kernel's): {dL/dcolor r, g, b, dL/ddepth, dL/dopacity, Sx, Sy, Sxx, Sxy, Syy, 0, 0}
with S.. = sum over pixels of u (dx, dy, dx^2, dx dy, dy^2), u = dL/dG * G, d = mean2D - pixel.

Error bound.  Next to every sum the reference returns a magnitude A (same sum with every signed inner sum replaced by
its sum of absolute values, each pair weighted by the error gain of its transmittance, see `_tile`).  A float32
implementation of the same operation is expected within EPS * A, for every Gaussian and component.  The model EPS
comes from, with u = 2^-24 (float32 unit roundoff) and g = 1 + M the pair's conic-form magnitude
(M = |A| dx^2 / 2 + |C| dy^2 / 2 + |B dx dy|, which bounds |power|):
  * power: five float32 operations on terms of size <= M: absolute error <= 3 u M, so G is off by a relative 3 u M;
  * G = ex2.approx(power * log2 e): 2^-22 relative (4 u), plus the rounding of the argument (u |power| <= u M);
    precise expf in the forward: 1 ulp.  Together with o G: alpha relative error <= 5 u g;
  * 1 - alpha: relative error <= u + 5 u g alpha / (1 - alpha) <= 5 u (1 + alpha g) / (1 - alpha);
  * T: the forward multiplies (1 - alpha) front to back and stores final_T; the backward recovers T_i by multiplying
    final_T with rcp.approx(1 - alpha) (1 ulp) back to front.  Each factor costs <= 10 u (1 + alpha_k g_k) /
    (1 - alpha_k), and T_i
    collects the factors of every contributor of its pixel (the forward's in front of i, both passes' behind i):
    relative error <= 20 u K with K = sum over the pixel's contributors of (1 + alpha_k g_k) / (1 - alpha_k) (the
    alpha error enters 1 - alpha scaled by alpha);
  * the pair's terms (w, dL/dalpha, u and the moments) add <= 10 rounding steps and one more alpha error (5 u g_i),
    each relative to the absolute-value form of the term: <= 15 u g_i + 20 u K + 10 u  <= 30 u (g_i + K);
  * float32 sums in any order (register sums, the shuffle butterfly, red.global across warps): <= (n - 1) u times the
    sum of absolute values for n summands; with gain >= 2 per pair, and n <= 100 red.global per Gaussian and
    component in the scenes tested, that is <= 50 u of A.
  Total 80 u = 4.8e-6.  EPS = 1e-5 is that, rounded up.

Ambiguity.  A pixel is flagged when a decision lies within float32 rounding of its threshold: alpha vs 1/255
(relative FLAG_TOL g), power vs 0 (FLAG_TOL M), T (1 - alpha) vs 1e-4 (relative T_TOL (1 + K)): `flag`; T vs 0.5
at the median crossing (relative T_TOL (1 + K)): `flag_median`.  `masked(upstream)` zeroes all four upstream images at
`flag` pixels and the median-depth image at `flag_median` pixels (that decision moves nothing but the median
gradient), so those pixels contribute nothing that depends on the decision, on either side: `sums` applies it, and a
GPU test applies it to its upstream.
"""
import numpy as np
import torch

F64 = torch.float64
TILE = 16
ALPHA_MIN = 1.0 / 255.0
ALPHA_MAX = 0.99
T_MIN = 1e-4
EPS = 1e-5
FLAG_TOL = 2e-6  # alpha vs 1/255 and power vs 0, relative to g and M: 6x the rounding of alpha and power
T_TOL = 2.5e-6   # T vs 1e-4 and 0.5, relative to 1 + K: 2x the 20 u K of the transmittance
LOG_NAMES = ("r", "g", "b", "depth", "opacity", "Sx", "Sy", "Sxx", "Sxy", "Syy")


def _t64(x):
    if x is None:
        return None
    if torch.is_tensor(x):
        return x.detach().to("cpu", F64)
    return torch.as_tensor(np.asarray(x), dtype=F64)


def _np(x, dtype):
    if torch.is_tensor(x):
        x = x.detach().cpu().numpy()
    return np.asarray(x, dtype=dtype)


def tile_lists(means2D, radii, depths, W, H, rect_dtype=np.float32):
    """Per-tile Gaussian lists from the tile rectangles of getRect (rasterizer auxiliary.h), evaluated in `rect_dtype`
    like the forward that produced means2D (float32 on the GPU), sorted by (float32 depth, index)."""
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    m = _np(means2D, rect_dtype).reshape(-1, 2)
    r = _np(radii, np.int64).reshape(-1)
    rr = r.astype(rect_dtype)
    t = rect_dtype(TILE)
    x0 = np.clip(np.trunc((m[:, 0] - rr) / t), 0, gx).astype(np.int64)
    y0 = np.clip(np.trunc((m[:, 1] - rr) / t), 0, gy).astype(np.int64)
    x1 = np.clip(np.trunc((m[:, 0] + rr + rect_dtype(TILE - 1)) / t), 0, gx).astype(np.int64)
    y1 = np.clip(np.trunc((m[:, 1] + rr + rect_dtype(TILE - 1)) / t), 0, gy).astype(np.int64)
    key = _np(depths, np.float32).reshape(-1)
    order = np.lexsort((np.arange(len(key)), key))  # by depth, ties by index
    lists = [[] for _ in range(gx * gy)]
    for i in order:
        if r[i] <= 0 or (x1[i] - x0[i]) * (y1[i] - y0[i]) == 0:
            continue
        for ty in range(y0[i], y1[i]):
            for tx in range(x0[i], x1[i]):
                lists[ty * gx + tx].append(int(i))
    return lists, gx, gy


class Compositing:
    """The geometry-only half of the reference for one forward: per-tile contributors, transmittances, flags and error
    gains.  `sums(upstream)` then gives the ten sums for any upstream images."""

    def __init__(self, means2D, conic_opacity, rgb, depths, radii, W, H, bg, rect_dtype=np.float32, lists=None):
        """lists: per-tile Gaussian lists to composite instead of the ones built here from the tile rectangles (a
        forward's own sorted list, when the question is what the compositing made of THAT list)."""
        self.W, self.H = int(W), int(H)
        self.m2 = _t64(means2D).reshape(-1, 2)
        self.co = _t64(conic_opacity).reshape(-1, 4)
        self.rgb = _t64(rgb).reshape(-1, 3)
        self.depth = _t64(depths).reshape(-1)
        self.bg = _t64(bg).reshape(3)
        self.P = self.m2.shape[0]
        self.gx, self.gy = (self.W + TILE - 1) // TILE, (self.H + TILE - 1) // TILE
        if lists is None:
            lists, _, _ = tile_lists(means2D, radii, depths, W, H, rect_dtype)
        assert len(lists) == self.gx * self.gy
        self.tiles = []
        HW = self.W * self.H
        self.flag = torch.zeros(HW, dtype=torch.bool)         # alpha, power or stop decision ambiguous
        self.flag_median = torch.zeros(HW, dtype=torch.bool)  # the median crossing ambiguous
        self.covered = torch.zeros(HW, dtype=torch.bool)
        self.n_contrib = torch.zeros(HW, dtype=torch.int64)   # contributors per pixel
        self.ended = torch.zeros(HW, dtype=torch.bool)        # the pixel ended on T < 1e-4
        self.final_T = torch.ones(HW, dtype=F64)
        self.median = torch.full((HW,), -1, dtype=torch.int64)  # Gaussian at which T crosses 0.5, -1: none
        self.last = torch.zeros(HW, dtype=torch.int64)  # 1 + list position of the last contributor (forward.cu's n_contrib)
        self.flag_kinds = {k: torch.zeros(HW, dtype=torch.bool) for k in ("alpha", "power", "stop", "median")}
        for t, ids in enumerate(lists):
            if ids:
                self.tiles.append(self._tile(t, torch.as_tensor(ids)))

    def _tile(self, t, ids):
        tx, ty = t % self.gx, t // self.gx
        k = torch.arange(TILE * TILE)
        px, py = tx * TILE + k % TILE, ty * TILE + k // TILE
        inside = (px < self.W) & (py < self.H)
        px, py = px[inside], py[inside]
        pid = py * self.W + px
        # pixel coordinates are the integer pixel indices, no +0.5 (forward.cu:343-344)
        dx = self.m2[ids, 0][None, :] - px.to(F64)[:, None]
        dy = self.m2[ids, 1][None, :] - py.to(F64)[:, None]
        A, B, C, o = (self.co[ids, j][None, :] for j in range(4))
        power = -0.5 * (A * dx * dx + C * dy * dy) - B * dx * dy
        Mterm = 0.5 * A.abs() * dx * dx + 0.5 * C.abs() * dy * dy + (B * dx * dy).abs()
        G = torch.exp(power)
        oG = o * G
        alpha = oG.clamp(max=ALPHA_MAX)
        valid = (power <= 0) & (alpha >= ALPHA_MIN)
        av = torch.where(valid, alpha, torch.zeros_like(alpha))
        incl = torch.cumprod(1 - av, dim=1)
        n = ids.numel()
        pos = torch.arange(n)[None, :]
        # the pixel ends at the first pair whose blend would take T below 1e-4; that pair does not blend
        ends = valid & (incl < T_MIN)
        kstop = torch.where(ends.any(1), ends.float().argmax(1), torch.full((pid.numel(),), n))
        contrib = valid & (pos < kstop[:, None])
        a = torch.where(contrib, alpha, torch.zeros_like(alpha))
        # T_i = prod_{k in front of i} (1 - alpha_k), a plain forward product
        T = torch.cumprod(torch.cat([torch.ones(pid.numel(), 1, dtype=F64), 1 - a], 1), dim=1)
        T_final, T = T[:, -1], T[:, :-1]
        Tnext = T * (1 - a)
        # the median-depth Gaussian: T > 0.5 in front of it and < 0.5 behind it (forward.cu:374-378)
        med = contrib & (T > 0.5) & (Tnext < 0.5)
        g = 1 + Mterm
        inv1a = 1 / (1 - a)
        K = torch.where(contrib, (1 + a * g) * inv1a, torch.zeros_like(g)).sum(1)
        gain = torch.where(contrib, g + K[:, None], torch.zeros_like(g))

        # ambiguity flags (only decisions that are taken matter: pairs up to and including the ending one)
        reach = pos <= kstop[:, None]
        f_alpha = (reach & (power <= 0) & ((oG / ALPHA_MIN - 1).abs() <= FLAG_TOL * g)).any(1)
        f_power = (reach & (Mterm > 0) & (power.abs() <= FLAG_TOL * Mterm) & (o >= ALPHA_MIN)).any(1)
        tolK = T_TOL * (1 + K)
        f_stop = (reach & valid & ((incl / T_MIN - 1).abs() <= tolK[:, None])).any(1)
        Ts = torch.cat([torch.where(contrib, T, torch.full_like(T, 10.0)), T_final[:, None]], 1)
        f_med = ((Ts / 0.5 - 1).abs() <= tolK[:, None]).any(1)
        for name, f in (("alpha", f_alpha), ("power", f_power), ("stop", f_stop), ("median", f_med)):
            self.flag_kinds[name][pid] = f
        self.flag[pid] = f_alpha | f_power | f_stop
        self.flag_median[pid] = f_med
        self.covered[pid] = contrib.any(1)
        self.n_contrib[pid] = contrib.sum(1)
        self.last[pid] = (contrib * (pos + 1)).max(1).values
        self.ended[pid] = kstop < n
        self.final_T[pid] = T_final
        has_med = med.any(1)
        self.median[pid[has_med]] = ids[med[has_med].float().argmax(1)]
        return dict(ids=ids, pid=pid, dx=dx, dy=dy, o=o, G=torch.where(contrib, G, torch.zeros_like(G)), T=T,
                    T_final=T_final, a=a, w=a * T, med=med, inv1a=inv1a, gain=gain, contrib=contrib,
                    stop_pos=kstop, oG=torch.where(contrib, oG, torch.zeros_like(oG)))

    def masked(self, dpix, ddepth, dmedian, dopacity):
        """The upstream images (torch or numpy, [3,H,W] and three [H,W]) with the ambiguous pixels zeroed."""
        keep = (~self.flag).reshape(self.H, self.W)
        keep_m = keep & (~self.flag_median).reshape(self.H, self.W)
        z = lambda x, k: torch.where(k, torch.as_tensor(x), torch.zeros((), dtype=torch.as_tensor(x).dtype))
        return z(dpix, keep), z(ddepth, keep), z(dmedian, keep_m), z(dopacity, keep)

    def sums(self, dpix, ddepth, dmedian, dopacity, drop_flagged=True):
        """-> (sums [P,12], A [P,12]) for the upstream images dpix [3,H,W], ddepth [H,W] and dmedian [H,W] (channel 0
        of the median-depth gradient) and dopacity [H,W]; drop_flagged: through `masked` first.
        Also sets self.reached: the Gaussians that contribute to a pixel with non-zero upstream."""
        if drop_flagged:
            dpix, ddepth, dmedian, dopacity = self.masked(dpix, ddepth, dmedian, dopacity)
        HW = self.W * self.H
        up = [_t64(x) for x in (dpix, ddepth, dmedian, dopacity)]
        gc = up[0].reshape(3, HW)
        gD = up[1].reshape(HW)
        gM = up[2].reshape(HW)  # channel 0 only (quirk 4)
        gO = up[3].reshape(HW)
        nz = (gc != 0).any(0) | (gD != 0) | (gM != 0) | (gO != 0)
        S = torch.zeros(self.P, 12, dtype=F64)
        Aall = torch.zeros(self.P, 12, dtype=F64)
        self.reached = torch.zeros(self.P, dtype=torch.bool)
        for tl in self.tiles:
            ids, pid = tl["ids"], tl["pid"]
            c = [gc[j, pid][:, None] for j in range(3)]
            d, m, op = gD[pid][:, None], gM[pid][:, None], gO[pid][:, None]
            rgb = [self.rgb[ids, j][None, :] for j in range(3)]
            dep = self.depth[ids][None, :]
            w, T, inv1a, G, o, dx, dy = tl["w"], tl["T"], tl["inv1a"], tl["G"], tl["o"], tl["dx"], tl["dy"]
            s = rgb[0] * c[0] + rgb[1] * c[1] + rgb[2] * c[2] + dep * d + op
            sabs = (rgb[0] * c[0]).abs() + (rgb[1] * c[1]).abs() + (rgb[2] * c[2]).abs() + (dep * d).abs() + op.abs()
            bgdot = sum(self.bg[j] * c[j][:, 0] for j in range(3))
            bgabs = sum((self.bg[j] * c[j][:, 0]).abs() for j in range(3))
            sw, swa = s * w, sabs * w
            # sum over the contributors behind each one (suffix sums), plus the background seen through T_final
            behind = sw.flip(1).cumsum(1).flip(1) - sw + (tl["T_final"] * bgdot)[:, None]
            behind_abs = swa.flip(1).cumsum(1).flip(1) - swa + (tl["T_final"] * bgabs)[:, None]
            dal = s * T - behind * inv1a
            dal_abs = sabs * T + behind_abs * inv1a
            ct = tl["contrib"]
            dal = torch.where(ct, dal, torch.zeros_like(dal))
            dal_abs = torch.where(ct, dal_abs, torch.zeros_like(dal_abs))
            # the median-depth gradient goes, whole, to the depth of the Gaussian at which T crosses 0.5
            medv = torch.where(tl["med"], m.expand_as(w), torch.zeros_like(w))
            # opacity: the gradient passes through the 0.99 clamp (dalpha/do = G even where alpha was clamped), and
            # the opacity image adds the direct term w gO on top of its share of dL/dalpha (quirk 5)
            u = o * G * dal
            ua = o * G * dal_abs
            terms = [w * c[0], w * c[1], w * c[2], w * d + medv, w * op + G * dal,
                     u * dx, u * dy, u * dx * dx, u * dx * dy, u * dy * dy]
            mags = [w * c[0].abs(), w * c[1].abs(), w * c[2].abs(), w * d.abs() + medv.abs(),
                    w * op.abs() + G * dal_abs,
                    ua * dx.abs(), ua * dy.abs(), ua * dx * dx, ua * (dx * dy).abs(), ua * dy * dy]
            gain = tl["gain"]
            self.reached[ids[(ct & nz[pid][:, None]).any(0)]] = True
            S[:, :10].index_add_(0, ids, torch.stack([x.sum(0) for x in terms], 1))
            Aall[:, :10].index_add_(0, ids, torch.stack([(x * gain).sum(0) for x in mags], 1))
        return S, Aall

    def stats(self):
        cov = int(self.covered.sum())
        return dict(covered=cov, flagged=int((self.flag & self.covered).sum()),
                    frac=float((self.flag & self.covered).sum()) / max(cov, 1),
                    median_frac=float((self.flag_median & self.covered).sum()) / max(cov, 1))


def to_upstream(S, conic_opacity, W, H):
    """Kernel 7's map of the sums to the per-Gaussian upstream of the projection (float64):
    dL/dmean2D = -(A Sx + B Sy, B Sx + C Sy) * (W/2, H/2), dL/dconic = -1/2 (Sxx, Sxy, Syy)."""
    S = _t64(S)
    co = _t64(conic_opacity).reshape(-1, 4)
    A, B, C = co[:, 0], co[:, 1], co[:, 2]
    m2 = torch.stack([-(A * S[:, 5] + B * S[:, 6]) * (0.5 * W), -(B * S[:, 5] + C * S[:, 6]) * (0.5 * H)], 1)
    return dict(mean2D=m2, conic=-0.5 * S[:, 7:10], color=S[:, 0:3], depth=S[:, 3], opacity=S[:, 4])


def to_upstream_abs(Am, conic_opacity, W, H):
    """The same map applied to the magnitudes: a bound on what the errors of the sums become."""
    Am = _t64(Am)
    co = _t64(conic_opacity).reshape(-1, 4).abs()
    A, B, C = co[:, 0], co[:, 1], co[:, 2]
    m2 = torch.stack([(A * Am[:, 5] + B * Am[:, 6]) * (0.5 * W), (B * Am[:, 5] + C * Am[:, 6]) * (0.5 * H)], 1)
    return dict(mean2D=m2, conic=0.5 * Am[:, 7:10], color=Am[:, 0:3], depth=Am[:, 3], opacity=Am[:, 4])


def worst_ratio(got, ref, Am, eps=EPS):
    """max over every Gaussian and component of |got - ref| / (eps A); -> (ratio, gaussian, component)."""
    got, ref, Am = _t64(got), _t64(ref), _t64(Am)
    e = (got - ref).abs()
    r = e / (eps * Am + 1e-300)
    r = torch.where(e == 0, torch.zeros_like(r), r)
    if not torch.isfinite(got).all():
        i = int((~torch.isfinite(got)).nonzero()[0, 0])
        return float("inf"), i, -1
    flat = int(r.argmax())
    return float(r.reshape(-1)[flat]), flat // r.shape[1], flat % r.shape[1]
