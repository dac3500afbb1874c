"""Float64 checks of the exact tile culling: the projection's tile mask (`tile_mask_of`, gsr_preprocess.cu) and the
rectangle test `may_touch` (gsr_internal.cuh), on the device's own float32 records promoted to float64.

A pair (Gaussian, pixel) contributes in the reference only if alpha = min(0.99, o exp(-q/2)) >= 1/255, i.e.
q(d) = A dx^2 + 2B dx dy + C dy^2 <= tau = 2 ln(255 o), d = pixel - mean, pixel coordinates the integer indices.

  coverage   every tile of a rect of <= 32 tiles with an in-image integer pixel where
             q64(d) <= tau64 + 1e-4 + 1e-6 S(d) (S = A dx^2 + C dy^2 + 2|B dx dy|, the pair's absolute term sum) has
             its bit set; o < 0.0039 gives an empty mask.  The slack is ~10x the float32 rounding of the reference's
             per-pixel test and ~10x below the kernel's own margin, so no pixel needs flagging.
  shape      no bit at or beyond the rect area; the mask is all ones where the kernel's guard fires (conic not positive
             definite or not finite, tau < 0, hx or hy >= 1e6), recomputed in float64 with a flag band around det = 0
             and hx, hy = 1e6.
  tightness  every set bit's pixel box x in [16tx, 16tx + 15], y in [16ty, min(16ty + 15, H - 1)], grown by 1 px,
             comes within taum * 1.001 of the kernel's margined threshold taum = tau + 1e-5 S_rect + 1e-3 (closed-form
             minimum of the convex q over the box).  The share of set bits with no qualifying integer pixel is
             reported.

The minimum of q - 1e-6 S over the integer pixels of one pixel row is exact: on each side of dx = 0 it is a convex
quadratic in x, so its integer minimum is the floor or the ceiling of its real minimiser clamped to the row's columns.

Also here: float32 restatements of tile_mask_of and may_touch (line for line, without FMA contraction) for the CPU
tests, the projection's float32 records (conic, radius, rect, tau) from a screen-space covariance, and the edge
families of Gaussians the culling has to survive."""
import numpy as np

TILE = 16
KBIG = 32
O_CUT = np.float32(0.0039)
SLACK_ABS, SLACK_REL = 1e-4, 1e-6
TIGHT = 1.001
# share of set bits with no qualifying integer pixel, per edge family: the float32 restatement's on the CPU families,
# rounded up.  The opacity family is mostly ellipses far below one pixel (tau ~ 0): the kernel's absolute margin 1e-3
# keeps their tile.  The Mip filter at kernel_size 0 leaves needles undilated, so most of their ellipses are thinner
# than a pixel row (restatement 0.78), and tiny ellipses tinier (0.95): MIP0_TIGHT_SHARE.  On the Mip path a singular
# or indefinite covariance gets coef 0 and so opacity 0 unless float32 rounding leaves det0 above 1e-6: the degenerate
# family there sets a handful of bits, too few for a share.
TIGHT_SHARE = {"needles": 0.2, "strips": 0.15, "boundaries": 0.2, "partial": 0.2, "opacity": 0.95, "rect32": 0.01,
               "degenerate": 0.3}
MIP0_TIGHT_SHARE = {k: v for k, v in dict(TIGHT_SHARE, needles=0.9, opacity=0.98).items() if k != "degenerate"}
f32 = np.float32


# ---- the projection's float32 records ---------------------------------------------------------------------------------
def tile_rect(px, py, radius, gx, gy):
    """auxiliary.h getRect in float32 (the (int) cast truncates toward zero)."""
    r = radius.astype(f32)
    t = lambda v, g: np.clip(np.trunc(np.nan_to_num(v, nan=0.0, posinf=1e9, neginf=-1e9)), 0, g).astype(np.int64)
    with np.errstate(all="ignore"):
        return (t((px - r) / f32(TILE), gx), t((py - r) / f32(TILE), gy),
                t((px + r + f32(TILE - 1)) / f32(TILE), gx), t((py + r + f32(TILE - 1)) / f32(TILE), gy))


def mip_input_opacity(cov, o, k):
    """The input opacity whose Mip-filtered opacity o coef (kernel_size k) is the wanted o (capped at 1), float64."""
    a, b, c = (np.asarray(v, np.float64) for v in cov)
    det0 = np.maximum(1e-6, a * c - b * b)
    det1 = np.maximum(1e-6, (a + k) * (c + k) - b * b)
    return np.minimum(np.asarray(o, np.float64) / np.sqrt(det0 / (det1 + 1e-6) + 1e-6), 1.0)


def records(px, py, cov, o, W, H, dil=0.3, mip=False):
    """The projection's float32 splat record from a screen-space covariance cov = (a, b, c) before the dilation:
    3DGS adds 0.3 to the diagonal; the Mip filter adds `dil` and scales o by its coef.  -> dict of px, py, A, B, C, o,
    tau (float32), radius, x0, y0, x1, y1 (int64)."""
    px, py, o = (np.asarray(v, f32) for v in (px, py, o))
    a, b, c = (np.asarray(v, f32) for v in cov)
    k = f32(dil)
    with np.errstate(all="ignore"):
        if mip:
            det0 = np.maximum(f32(1e-6), a * c - b * b)
            det1 = np.maximum(f32(1e-6), (a + k) * (c + k) - b * b)
            coef = np.where((det0 <= f32(1e-6)) | (det1 <= f32(1e-6)), f32(0),
                            np.sqrt(det0 / (det1 + f32(1e-6)) + f32(1e-6))).astype(f32)
            o = (o * coef).astype(f32)
        cx, cy, cz = a + k, b, c + k
        det = cx * cz - cy * cy
        di = f32(1) / det
        A, B, C = cz * di, -cy * di, cx * di
        mid = f32(0.5) * (cx + cz)
        l1 = mid + np.sqrt(np.maximum(f32(0.1), mid * mid - det))
        l2 = mid - np.sqrt(np.maximum(f32(0.1), mid * mid - det))
        rad = np.ceil(f32(3) * np.sqrt(np.maximum(l1, l2)))
        rad = np.where(np.isfinite(rad) & (det != 0), rad, 0).astype(np.int64)
        tau = (f32(2) * np.log(f32(255) * o)).astype(f32)
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    x0, y0, x1, y1 = tile_rect(px, py, rad, gx, gy)
    live = (rad > 0) & ((x1 - x0) * (y1 - y0) > 0)
    return dict(px=px, py=py, A=A.astype(f32), B=B.astype(f32), C=C.astype(f32), o=o, tau=tau, radius=rad,
                x0=np.where(live, x0, 0), y0=np.where(live, y0, 0), x1=np.where(live, x1, 0), y1=np.where(live, y1, 0),
                W=W, H=H)


# ---- float32 restatement of tile_mask_of (CPU tests only) --------------------------------------------------------------
def tile_mask_f32(r, margins=True, extent_margins=True, hclamp=None):
    """tile_mask_of line for line in float32 on records `r`; masks [N] int64.  margins=False drops every margin of the
    kernel (the x-extent's 1.0001 and 0.01 px, and taum's 1e-5 S + 1e-3), extent_margins=False only the x-extent's;
    hclamp: the row band's clamp (H - 1 in the kernel).  Rects of more than 32 tiles get all ones (the kernel does not compute a mask for them)."""
    px, py, A, B, C, o, tau = (r[k] for k in ("px", "py", "A", "B", "C", "o", "tau"))
    x0, y0, x1, y1 = (r[k] for k in ("x0", "y0", "x1", "y1"))
    H = r["H"]
    hcl = H - 1 if hclamp is None else hclamp
    rw = x1 - x0
    n = rw * (y1 - y0)
    allm = np.where(n >= 32, 0xffffffff, (np.int64(1) << np.minimum(n, 32)) - 1)
    with np.errstate(all="ignore"):
        det = A * C - B * B
        ok = (A > f32(1e-30)) & (C > f32(1e-30)) & (det > 0) & (A < f32(1e30)) & (C < f32(1e30)) & (tau >= 0)
        mx = np.maximum(np.abs(px - (x0 * TILE).astype(f32)), np.abs((x1 * TILE).astype(f32) - px))
        my = np.maximum(np.abs(py - (y0 * TILE).astype(f32)), np.abs((y1 * TILE).astype(f32) - py))
        taum = tau + f32(1e-5) * (A * mx * mx + C * my * my + f32(2) * np.abs(B) * mx * my) + f32(1e-3)
        taum = taum if margins else tau
        idet, iA = f32(1) / det, f32(1) / A
        hx, hy = np.sqrt(taum * C * idet), np.sqrt(taum * A * idet)
        ok &= (hx < f32(1e6)) & (hy < f32(1e6))
        dyx = -B * hx / C
        D, BA = det * iA, B * iA
        mask = np.zeros(len(px), np.int64)
        m1, a1 = (f32(1.0001), f32(0.01)) if margins and extent_margins else (f32(1), f32(0))
        for k in range(KBIG):
            ty = y0 + k
            row = ok & (ty < y1)
            lo = np.maximum((ty * TILE).astype(f32) - py, -hy)
            hi = np.minimum(np.minimum(ty * TILE + TILE - 1, hcl).astype(f32) - py, hy)
            row &= ~(lo > hi)
            da = np.minimum(np.maximum(dyx, lo), hi)
            db = np.minimum(np.maximum(-dyx, lo), hi)
            xmax = -BA * da + np.sqrt(np.maximum(f32(0), (taum - D * da * da) * iA)) * m1 + a1
            xmin = -BA * db - np.sqrt(np.maximum(f32(0), (taum - D * db * db) * iA)) * m1 - a1
            fin = lambda v: np.nan_to_num(v, nan=0.0, posinf=1e9, neginf=-1e9)
            ta = np.maximum(x0, fin(np.ceil((px + xmin - f32(TILE - 1)) * f32(1.0 / TILE))).astype(np.int64))
            tb = np.minimum(x1 - 1, fin(np.floor((px + xmax) * f32(1.0 / TILE))).astype(np.int64))
            row &= ta <= tb
            first = np.clip(k * rw + (ta - x0), 0, 63)
            ln = np.clip(tb - ta + 1, 0, 32)
            bits = (((np.int64(1) << ln) - 1) << first) & 0xffffffff
            mask |= np.where(row, bits, 0)
    mask = np.where(ok, mask, allm) & allm
    mask = np.where(o < O_CUT, 0, mask)
    return np.where(n > KBIG, 0xffffffff, mask)


def may_touch_f32(gx, gy, A, B, C, o, tau, rx0, ry0, rx1, ry1):
    """may_touch (cull_prep + the rectangle test) in float32; exact reciprocals where the kernel takes rcp.approx."""
    gx, gy, A, B, C, o, tau = (np.asarray(v, f32) for v in (gx, gy, A, B, C, o, tau))
    rx0, ry0, rx1, ry1 = (np.asarray(v, f32) for v in (rx0, ry0, rx1, ry1))
    with np.errstate(all="ignore"):
        odd = ~((A > f32(1e-30)) & (C > f32(1e-30)) & (A * C - B * B > 0) & (A < f32(1e30)) & (C < f32(1e30)))
        nBiC, nBiA = -B * (f32(1) / C), -B * (f32(1) / A)
        dxlo, dxhi, dylo, dyhi = gx - rx1, gx - rx0, gy - ry1, gy - ry0
        inx, iny = (dxlo <= 0) & (dxhi >= 0), (dylo <= 0) & (dyhi >= 0)
        dxe = np.where(dxlo > 0, dxlo, dxhi)
        dys = np.minimum(np.maximum(nBiC * dxe, dylo), dyhi)
        q1 = A * dxe * dxe + f32(2) * B * dxe * dys + C * dys * dys
        dye = np.where(dylo > 0, dylo, dyhi)
        dxs = np.minimum(np.maximum(nBiA * dye, dxlo), dxhi)
        q2 = A * dxs * dxs + f32(2) * B * dxs * dye + C * dye * dye
        qmin = np.minimum(np.where(inx, f32(3e38), q1), np.where(iny, f32(3e38), q2))
        mx, my = np.maximum(np.abs(dxlo), np.abs(dxhi)), np.maximum(np.abs(dylo), np.abs(dyhi))
        S = A * mx * mx + C * my * my + f32(2) * np.abs(B) * mx * my
        keep = (inx & iny) | odd | ~(qmin > tau + f32(1e-5) * S + f32(1e-3))
    return keep & ~(o < O_CUT)


# ---- float64 pieces ---------------------------------------------------------------------------------------------------
def _d(r, *keys):
    return tuple(np.asarray(r[k], np.float64) for k in keys)


def block_qmin(px, py, A, B, C, bx, by, bw, bh, W, H, eps=SLACK_REL):
    """Over the in-image integer pixels of the blocks [bx, bx + bw) x [by, by + bh) (arrays [N, K] of block origins;
    px .. C [N]): -> (min of q, min of q - eps S), float64 [N, K]; +inf for blocks with no in-image pixel."""
    N, K = bx.shape
    sh = lambda v: v[:, None, None]
    px_, py_, A_, B_, C_ = sh(px), sh(py), sh(A), sh(B), sh(C)
    y = by[:, :, None] + np.arange(bh)[None, None, :]            # [N, K, bh]
    xlo = bx[:, :, None].astype(np.float64) + 0 * y
    xhi = np.minimum(bx[:, :, None] + bw - 1, W - 1).astype(np.float64) + 0 * y
    valid = (y < H) & (xlo <= xhi)
    dy = y - py_
    Bdy = B_ * dy
    qbest = np.full(y.shape, np.inf)
    gbest = np.full(y.shape, np.inf)
    with np.errstate(all="ignore"):
        cands = [px_ - Bdy / A_]
        for s in (1.0, -1.0):
            cands.append(px_ - (Bdy - s * eps * np.abs(Bdy)) / ((1 - eps) * A_))
        for c in cands:
            c = np.clip(np.nan_to_num(c, nan=0.0), xlo, xhi)
            for x in (np.floor(c), np.ceil(c)):
                x = np.clip(x, xlo, xhi)
                dx = x - px_
                q = A_ * dx * dx + 2 * Bdy * dx + C_ * dy * dy
                S = A_ * dx * dx + C_ * dy * dy + 2 * np.abs(Bdy * dx)
                qbest = np.minimum(qbest, q)
                gbest = np.minimum(gbest, q - eps * S)
    qbest = np.where(valid, qbest, np.inf)
    gbest = np.where(valid, gbest, np.inf)
    return qbest.min(2), gbest.min(2)


def box_qmin(px, py, A, B, C, x0, y0, x1, y1):
    """float64 minimum of the convex q over the real boxes [x0, x1] x [y0, y1] (arrays of one shape)."""
    with np.errstate(all="ignore"):
        dxl, dxh, dyl, dyh = x0 - px, x1 - px, y0 - py, y1 - py
        inside = (dxl <= 0) & (dxh >= 0) & (dyl <= 0) & (dyh >= 0)
        best = np.full(np.broadcast(px, x0).shape, np.inf)
        for dx in (dxl, dxh):
            dy = np.clip(-B * dx / C, dyl, dyh)
            best = np.minimum(best, A * dx * dx + 2 * B * dx * dy + C * dy * dy)
        for dy in (dyl, dyh):
            dx = np.clip(-B * dy / A, dxl, dxh)
            best = np.minimum(best, A * dx * dx + 2 * B * dx * dy + C * dy * dy)
    return np.where(inside, 0.0, best)


def _taum64(r):
    """The kernel's margined threshold and its rect-wide term sum, in float64."""
    px, py, A, B, C, tau = _d(r, "px", "py", "A", "B", "C", "tau")
    x0, y0, x1, y1 = (np.asarray(r[k], np.float64) * TILE for k in ("x0", "y0", "x1", "y1"))
    mx = np.maximum(np.abs(px - x0), np.abs(x1 - px))
    my = np.maximum(np.abs(py - y0), np.abs(y1 - py))
    with np.errstate(all="ignore"):
        S = A * mx * mx + C * my * my + 2 * np.abs(B) * mx * my
    return tau + 1e-5 * S + 1e-3


def guard64(r):
    """The kernel's keep-everything guard recomputed in float64 -> (fires, flagged): flagged where float32 rounding of
    det, hx or hy could decide it either way."""
    A, B, C, tau = _d(r, "A", "B", "C", "tau")
    with np.errstate(all="ignore"):
        det = A * C - B * B
        fin = np.isfinite(A) & np.isfinite(B) & np.isfinite(C) & np.isfinite(tau)
        basic = ~((A > 1e-30) & (C > 1e-30) & (A < 1e30) & (C < 1e30) & (tau >= 0) & fin)
        det_flag = np.abs(det) <= 1e-5 * (np.abs(A * C) + B * B)
        taum = _taum64(r)
        hx, hy = np.sqrt(taum * C / det), np.sqrt(taum * A / det)
        big = ~((hx < 1e6) & (hy < 1e6)) | ~np.isfinite(taum)
        h_flag = (np.abs(hx / 1e6 - 1) <= 1e-3) | (np.abs(hy / 1e6 - 1) <= 1e-3)
        fires = basic | (det <= 0) | big
        flag = ~basic & (det_flag | h_flag)
    return fires, flag


def _bits(r):
    """-> (area [N], rect width [N], tile x / y of every bit [N, 32], bit exists [N, 32])."""
    x0, y0, x1, y1 = (np.asarray(r[k], np.int64) for k in ("x0", "y0", "x1", "y1"))
    w = np.maximum(x1 - x0, 0)
    n = w * np.maximum(y1 - y0, 0)
    i = np.arange(KBIG)[None, :]
    ws = np.maximum(w, 1)[:, None]
    return n, w, x0[:, None] + i % ws, y0[:, None] + i // ws, i < n[:, None]


# ---- the checks -------------------------------------------------------------------------------------------------------
class Report:
    """What check_mask found: `errors` per check (lists of (gaussian, message)), and the measured numbers."""

    def __init__(self):
        self.errors = {"coverage": [], "shape": [], "tightness": []}
        self.stats = {}

    def fail(self, check, rows, msg):
        for i in np.atleast_1d(rows)[:5]:
            self.errors[check].append((int(i), msg(int(i))))
        if len(np.atleast_1d(rows)) > 5:
            self.errors[check].append((-1, f"... {len(np.atleast_1d(rows))} Gaussians in all"))

    def failed(self):
        return {k for k, v in self.errors.items() if v}

    def text(self):
        return "; ".join(f"{k}: " + ", ".join(m for _, m in v) for k, v in self.errors.items() if v)


def check_mask(r, mask, chunk=1000):
    """Coverage, shape and tightness of `mask` [N] (uint32 as int64) for the float32 records `r` (dict as `records`
    returns, or read from a geometry buffer).  -> Report with stats: worst coverage slack (the smallest fraction of the
    kernel's margin taum - tau left over a pixel of a required tile), tightness share, fallback count, and counts."""
    rep = Report()
    mask = np.asarray(mask, np.int64) & 0xffffffff
    n, w, tx, ty, exists = _bits(r)
    px, py, A, B, C, o, tau = _d(r, "px", "py", "A", "B", "C", "o", "tau")
    W, H = int(r["W"]), int(r["H"])
    small = (n > 0) & (n <= KBIG)
    bit = ((mask[:, None] >> np.arange(KBIG)[None, :]) & 1).astype(bool)
    allm = np.where(n >= 32, 0xffffffff, (np.int64(1) << np.minimum(n, 32)) - 1)
    dead = o < float(O_CUT)
    fires, flag = guard64(r)
    with np.errstate(all="ignore"):
        tau64 = 2 * np.log(255 * o)
        taum = _taum64(r)
    # shape
    bad = small & (mask & ~allm & 0xffffffff != 0)
    rep.fail("shape", np.nonzero(bad)[0], lambda i: f"#{i} has bits beyond its rect area {n[i]} (mask {mask[i]:#x})")
    bad = small & dead & (mask != 0)
    rep.fail("shape", np.nonzero(bad)[0], lambda i: f"#{i} has o = {o[i]:.9g} < 0.0039 but mask {mask[i]:#x}")
    bad = small & ~dead & fires & ~flag & (mask != allm)
    rep.fail("shape", np.nonzero(bad)[0], lambda i: f"#{i}: the guard fires (A {A[i]:.6g} B {B[i]:.6g} C {C[i]:.6g} "
                                                     f"tau {tau[i]:.6g}) but mask {mask[i]:#x} != {allm[i]:#x}")
    # coverage and tightness on the Gaussians that compute a mask
    with np.errstate(all="ignore"):
        pd = np.isfinite(A) & np.isfinite(B) & np.isfinite(C) & (A > 0) & (A * C - B * B > 0)
    cov_rows = np.nonzero(small & ~dead & pd)[0]
    slack_min, n_req, n_set, n_loose = np.inf, 0, 0, 0
    worst_tight = 0.0
    for s in range(0, len(cov_rows), chunk):
        g = cov_rows[s:s + chunk]
        qmin, gmin = block_qmin(px[g], py[g], A[g], B[g], C[g], tx[g] * TILE, ty[g] * TILE, TILE, TILE, W, H)
        req = exists[g] & (gmin <= (tau64[g] + SLACK_ABS)[:, None])
        miss = req & ~bit[g]
        rows = g[miss.any(1)]
        rep.fail("coverage", rows, lambda i: f"#{i} (px {px[i]:.9g} py {py[i]:.9g} A {A[i]:.9g} B {B[i]:.9g} C "
                                             f"{C[i]:.9g} o {o[i]:.9g}) rect {n[i]} tiles, mask {mask[i]:#x}: a "
                                             f"required tile is not binned")
        n_req += int(req.sum())
        if req.any():
            sl = (taum[g][:, None] - qmin) / (taum[g] - tau64[g])[:, None]
            slack_min = min(slack_min, float(sl[req].min()))
        # tightness: Gaussians the guard certainly passes
        t = ~(fires[g] | flag[g])
        setb = exists[g] & bit[g] & t[:, None]
        bx0, by0 = tx[g] * TILE - 1.0, ty[g] * TILE - 1.0
        bx1 = tx[g] * TILE + TILE * 1.0
        by1 = np.minimum(ty[g] * TILE + TILE - 1, H - 1) + 1.0
        sh = lambda v: v[:, None]
        qb = box_qmin(sh(px[g]), sh(py[g]), sh(A[g]), sh(B[g]), sh(C[g]), bx0, by0, bx1, by1)
        ratio = qb / sh(taum[g] * TIGHT)
        loose = setb & ~(ratio <= 1)
        rep.fail("tightness", g[loose.any(1)], lambda i: f"#{i} (px {px[i]:.9g} py {py[i]:.9g} A {A[i]:.9g} B "
                                                         f"{B[i]:.9g} C {C[i]:.9g}) mask {mask[i]:#x}: a set bit's "
                                                         f"box is beyond taum * {TIGHT}")
        if setb.any():
            worst_tight = max(worst_tight, float(np.where(setb, ratio * TIGHT, 0).max()))
        n_set += int(setb.sum())
        n_loose += int((setb & ~req).sum())
    rep.stats = dict(n=int(len(mask)), masked=int(small.sum()), checked=int(len(cov_rows)), required=n_req,
                     set=n_set, slack_min=float(slack_min), tight_share=n_loose / max(n_set, 1),
                     worst_tight=worst_tight, fallback=int((small & ~dead & fires).sum()),
                     flagged=int((small & ~dead & flag).sum()), dead=int((small & dead).sum()))
    return rep


def check_may_touch(r, bw, bh, K=32, seed=0, chunk=2000):
    """may_touch on K blocks of bw x bh per Gaussian, placed at random over the ellipse's bounding box grown by two
    blocks: -> (n blocks that need the Gaussian but may_touch drops, share of kept blocks with no qualifying pixel,
    number of needed blocks)."""
    rng = np.random.RandomState(seed)
    px, py, A, B, C, o = _d(r, "px", "py", "A", "B", "C", "o")
    N = len(px)
    with np.errstate(all="ignore"):
        tau64 = 2 * np.log(255 * o)
        det = A * C - B * B
        t = np.maximum(tau64, 0) + 1
        hx = np.nan_to_num(np.sqrt(t * C / det), nan=64, posinf=64)
        hy = np.nan_to_num(np.sqrt(t * A / det), nan=64, posinf=64)
    hx, hy = np.minimum(hx, 4096) + 2 * bw, np.minimum(hy, 4096) + 2 * bh
    bx = np.floor((px[:, None] + (2 * rng.rand(N, K) - 1) * hx[:, None]) / bw) * bw
    by = np.floor((py[:, None] + (2 * rng.rand(N, K) - 1) * hy[:, None]) / bh) * bh
    keep = may_touch_f32(r["px"][:, None], r["py"][:, None], r["A"][:, None], r["B"][:, None], r["C"][:, None],
                         r["o"][:, None], r["tau"][:, None], bx, by, bx + bw - 1, by + bh - 1)
    miss, kept, loose, need = 0, 0, 0, 0
    with np.errstate(all="ignore"):
        pd = (A > 0) & (det > 0) & np.isfinite(det)
    for s in range(0, N, chunk):
        g = np.arange(s, min(N, s + chunk))
        g = g[pd[g]]
        _, gmin = block_qmin(px[g], py[g], A[g], B[g], C[g], bx[g].astype(np.int64), by[g].astype(np.int64), bw, bh,
                             1 << 30, 1 << 30)
        req = (gmin <= (tau64[g] + SLACK_ABS)[:, None]) & (o[g] >= float(O_CUT))[:, None]
        miss += int((req & ~keep[g]).sum())
        kept += int(keep[g].sum())
        loose += int((keep[g] & ~req).sum())
        need += int(req.sum())
    return miss, loose / max(kept, 1), need


# ---- edge families (screen space) -------------------------------------------------------------------------------------
IMAGES = {"1x1": (1, 1), "17x9": (17, 9), "250x170": (250, 170), "1920x1080": (1920, 1080), "8192x4608": (8192, 4608)}
FAMILIES = ("needles", "strips", "boundaries", "partial", "opacity", "rect32", "degenerate")


def _rot(theta, l1, l2):
    c, s = np.cos(theta), np.sin(theta)
    return c * c * l1 + s * s * l2, c * s * (l1 - l2), s * s * l1 + c * c * l2


def family(name, n, W, H, seed=0, dil=0.3):
    """n Gaussians of one edge family on a W x H image: dict px, py, cov (a, b, c before the dilation), o (float64);
    `dil` is the dilation the covariance will get (0.3, or the Mip filter's width).  Families:
      needles     major variance 1 .. 2e4 px^2, minor 0 .. 1e-3 (the condition number the dilation allows), every
                  orientation with B = 0 and 45 degrees exactly among them;
      strips      huge Gaussians centred 5000 px beyond a border or a corner, their clipped rect a strip or a corner;
      boundaries  centres on tile and pixel boundaries (16k, 16k + 15, .5, +- 1e-3);
      partial     centres near the right and bottom edges, the last tiles partial;
      opacity     o at the 0.0039 cut and at 1/255 +- a few ulps (tau ~ 0, a tiny ellipse), and just above;
      rect32      rects of 32 and 33 tiles: 4x8, 8x4, 32x1, 1x32, 33x1 (off a corner or a border);
      degenerate  indefinite and singular covariances."""
    rng = np.random.RandomState(seed)
    u = lambda lo, hi: rng.uniform(lo, hi, n)
    px, py = u(-8, W + 8), u(-8, H + 8)
    o = rng.uniform(0.0039, 1.0, n)
    th = rng.uniform(0, np.pi, n)
    l1 = np.exp(u(np.log(0.05), np.log(200.0)))
    l2 = np.exp(u(np.log(0.05), np.log(200.0)))
    if name == "needles":
        th[::7], th[1::7], th[2::7] = 0.0, np.pi / 4, np.pi / 2
        l1 = np.exp(u(0, np.log(2e4)))
        l2 = np.where(rng.rand(n) < 0.5, 0.0, u(0, 1e-3))
        o = np.exp(u(np.log(0.004), 0))
    elif name == "strips":
        off = 5000.0
        side = rng.randint(0, 8, n)  # 0-3 borders, 4-7 corners
        px = np.where(side == 0, -off, np.where(side == 1, W + off, u(0, W)))
        py = np.where(side == 2, -off, np.where(side == 3, H + off, u(0, H)))
        cx, cy = np.where(side % 2 == 0, -off, W + off), np.where(side < 6, -off, H + off)
        px, py = np.where(side >= 4, cx, px), np.where(side >= 4, cy, py)
        # long axis toward the image; the radius 3 sigma reaches 0 .. 60 px into it and so does the ellipse (o >= 0.5)
        th = np.arctan2(H / 2 - py, W / 2 - px) + rng.normal(0, 0.02, n)
        reach = np.maximum(np.where(px < 0, -px, np.maximum(px - W + 1, 0)), np.where(py < 0, -py, np.maximum(py - H + 1, 0)))
        o = rng.uniform(0.5, 1.0, n)
        l1 = ((reach + u(0, 60)) / 3) ** 2
        l2 = l1 * u(1e-4, 0.5)
    elif name == "boundaries":
        bxs = np.array([0.0, 15.0, 0.5, 15.5, 1e-3, -1e-3, 16 - 1e-3, 7.5, 8.0])
        px = TILE * rng.randint(0, max(1, (W + 15) // 16), n) + rng.choice(bxs, n)
        py = TILE * rng.randint(0, max(1, (H + 15) // 16), n) + rng.choice(bxs, n)
    elif name == "partial":
        px = np.where(rng.rand(n) < 0.6, W - 1 + u(-6, 6), px)
        py = np.where(rng.rand(n) < 0.6, H - 1 + u(-6, 6), py)
        l1, l2 = l1 / 10, l2 / 10
    elif name == "opacity":
        base = np.float32(1 / 255)
        ulps = rng.randint(-4, 5, n).astype(np.float32)
        o32 = base + ulps * (np.nextafter(base, np.float32(1)) - base)
        pick = rng.rand(n)
        o = np.where(pick < 0.2, np.float32(0.0039) + rng.randint(-3, 4, n) * np.float32(2.3283064e-10),
                     np.where(pick < 0.7, o32, 1 / 255 * (1 + np.exp(u(np.log(1e-6), np.log(1.0))))))
        l1, l2 = l1 / 20, l2 / 20
    elif name == "rect32":
        gx, gy = (W + 15) // 16, (H + 15) // 16
        shape = rng.randint(0, 5, n)
        # radius r puts the far rect edge near 16 k tiles from the clipped border
        want = np.array([[4, 8], [8, 4], [32, 1], [1, 32], [33, 1]])[shape]
        r = np.maximum(want[:, 0], want[:, 1]) * 16.0 / 2 + u(-10, 10)
        # off a corner: the rect spans [0, (px + r)/16) x [0, (py + r)/16)
        px = want[:, 0] * 16.0 - r + u(-14, 2)
        py = want[:, 1] * 16.0 - r + u(-14, 2)
        px = np.where(want[:, 0] >= gx, u(0, W), px)
        py = np.where(want[:, 1] >= gy, u(0, H), py)
        lam = (r / 3) ** 2 - dil
        ratio = u(0.02, 1.0)
        l1, l2 = np.maximum(lam, 0.05), np.maximum(lam * ratio, 0.0)
    elif name == "degenerate":
        k = rng.randint(0, 3, n)
        l2 = np.where(k == 0, -dil * u(0.2, 3.0), np.where(k == 1, -dil, -dil * (1 + 1e-7)))
        l1 = np.abs(l1) + 1
    cov = _rot(th, l1, l2)
    return dict(px=px, py=py, cov=cov, o=o)
