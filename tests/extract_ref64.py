"""Float64 restatements of the extraction kernels' contracts, with the error bound each kernel must meet.

The contract is the reference script's (gaustudio/scripts/extract_pcd.py and Camera.depth2point / depth2normal), in
real numbers, evaluated in float64 on the float32 inputs:

  bilateral64      masked bilateral filter: dilation of the invalid mask (pixels outside the image never invalidate a
                   window), min / max over valid non-NaN depths in the kernel's order-preserving key order (-0 < +0),
                   normalisation with invalid pixels at 0, disc support r_ij <= r with centre weight 1 and the host's
                   float32 space weights, range weight exp(diff^2 * gc) evaluated directly (not OpenCV's 4096-bin
                   table), OpenCV's REFLECT_101 with repeated reflection, de-normalisation, masked-out pixels restored.
  depth2point64    Camera.depth2point with integer pixel coordinates (NaN coordinates for a 1-wide / 1-high map, as
                   the reference's u / (W - 1) gives), optional cam_to_world.
  depth2normal64   the 5-point cross normal -normalize(cross(top - bottom, left - right)), eps 1e-12, -1 fill on the
                   border and where a depth is outside (dmin, dmax), optional rotation.
  view_normals64   extract_pcd.py:325-335: the normals of depth2normal64, -1 fill outside the mask, the rotation
                   applied to the fill as well, validity sum(fill @ rot) > -3 & median < 0.8 radius & opacity > 0.5.
  fusion64         both passes of normal_fusion with the weight conf * |dot(v/|v|, n)| / (|v| + 1e-6), the strict
                   |n - mean| < 0.8 test against pass 1's mean, ids outside [0, P) skipped, F.normalize (NaN where the
                   weight is 0), and the smoothing over the k nearest points.
  knn64            exact float64 squared distances of the float32 points, ordered by (distance, index).

Error model.  Every output element must satisfy |gpu - ref| <= EPS * A, EPS = 2u with u = 2^-24, the float32 unit
roundoff.  A is the first-order error of the kernel's float32 evaluation in units of u: the sum of the magnitudes of
the terms that make up the value, each weighted by its error gain.  The factor 2 covers the second-order terms.  The
gains count:
  * one u per correctly rounded operation (the kernels' explicit __fmul_rn / __fadd_rn / __fdiv_rn, IEEE division
    and sqrtf; nvcc's FMA contraction under -fmad=true only removes roundings, so the count stays an upper bound);
  * 4u relative for expf (CUDA's expf is within 2 ulp, and one ulp is at most 2u relative);
  * (m - 1) u * sum |terms| for a sum of m terms added in any order, which covers the red.global.add sums of the
    fusion and the fixed-order window sums of the filter;
  * the conditioning of a cross product, a dot product and a normalisation: an input error e moves |c| / |sum| by
    e / |sum|, so a value made of terms that cancel gets a bound of sum |terms| / |sum terms| times their error.
Decisions are exact when their inputs are the same float32 values (the masks, (dmin, dmax), the fill, median and
opacity tests); a decision on a computed value is compared with the float64 value, and an element whose float64 value
lies within its own bound of the threshold is flagged instead (the 0.8 consistency test, the k-th neighbour cut).
"""
import numpy as np

from oracle.extract_oracle import reflect101  # OpenCV's BORDER_REFLECT_101, repeated; 0 when the side is 1 pixel

U = 2.0 ** -24
EPS = 2 * U
f32 = np.float32


class CheckError(AssertionError):
    pass


def fail(check, msg):
    raise CheckError(f"{check}: {msg}")


def close(check, got, ref, A, report=None):
    """|got - ref| <= EPS * A element by element, NaN exactly where ref is NaN; returns the worst err / bound."""
    got = np.asarray(got, np.float64)
    ref = np.asarray(ref, np.float64)
    A = np.broadcast_to(np.asarray(A, np.float64), ref.shape)
    if got.shape != ref.shape:
        fail(check, f"shape {got.shape} != {ref.shape}")
    if not np.array_equal(np.isnan(got), np.isnan(ref)):
        bad = np.argwhere(np.isnan(got) != np.isnan(ref))
        fail(check, f"NaN pattern differs at {len(bad)} elements, first {tuple(bad[0])}")
    ok = ~np.isnan(ref)
    inf = ok & np.isinf(ref)
    if not np.array_equal(got[inf], ref[inf]):
        fail(check, "infinite values differ")
    fin = ok & ~inf
    err = np.abs(got[fin] - ref[fin])
    bound = EPS * A[fin]
    if (err > bound).any():
        i = int(np.argmax(err - bound))
        at = tuple(np.argwhere(fin)[i])
        fail(check, f"|gpu - ref| = {err[i]:.3e} > bound {bound[i]:.3e} at {at} (gpu {got[fin][i]!r}, ref {ref[fin][i]!r})")
    worst = float(np.max(err / np.maximum(bound, 1e-300))) if err.size else 0.0
    if report is not None:
        report[check] = max(report.get(check, 0.0), worst)
    return worst


def exact(check, got, ref):
    got, ref = np.asarray(got), np.asarray(ref)
    if got.shape != ref.shape or not np.array_equal(got, ref):
        n = int((got != ref).sum()) if got.shape == ref.shape else -1
        fail(check, f"not identical ({n} elements differ)")


def same_bits(check, got, ref):
    """float32 arrays identical bit for bit (NaN payloads and -0.0 included)."""
    exact(check, np.asarray(got, f32).view(np.uint32), np.asarray(ref, f32).view(np.uint32))


# ---- masked bilateral filter ----------------------------------------------------------------------------------------
def f2key(x):
    """The kernel's order-preserving float -> uint32 key (atomicMin / atomicMax order the floats, -0.0 < +0.0)."""
    b = np.asarray(x, f32).view(np.uint32)
    return np.where(b & 0x80000000, ~b, b | 0x80000000).astype(np.uint32)


def key2f(k):
    k = np.asarray(k, np.uint32)
    return np.where(k & 0x80000000, k & 0x7fffffff, ~k).astype(np.uint32).view(f32)


def space_weights(r, sigma_space):
    """(dy, dx, w) of the disc r_ij <= r without the centre, w the host's float32 (float)exp(rr^2 * gs) from double."""
    ss = float(f32(sigma_space))
    ss = 1.0 if ss <= 0 else ss
    gs = -0.5 / (ss * ss)
    out = []
    for dy in range(-r, r + 1):
        for dx in range(-r, r + 1):
            rr = np.sqrt(float(dy * dy + dx * dx))
            if rr > r or (dy == 0 and dx == 0):
                continue
            out.append((dy, dx, float(f32(np.exp(rr * rr * gs)))))
    return out


def dilated_mask(mask, r):
    H, W = mask.shape
    inv = np.zeros((H + 2 * r, W + 2 * r), bool)  # pixels outside the image never invalidate a window
    inv[r:r + H, r:r + W] = ~mask
    dil = np.zeros((H, W), bool)
    for dy in range(2 * r + 1):
        for dx in range(2 * r + 1):
            dil |= inv[dy:dy + H, dx:dx + W]
    return ~dil


def bilateral64(depth, mask, d=3, sigma_color=75.0, sigma_space=75.0):
    """-> dict(filtered [H,W] f64, A [H,W], new_mask, valid, vmin, vmax (float32 or None))."""
    depth = np.asarray(depth, f32)
    mask = np.asarray(mask, bool)
    H, W = depth.shape
    r = d // 2
    new_mask = dilated_mask(mask, r)
    valid = new_mask & ~np.isnan(depth)
    out = depth.astype(np.float64)
    A = np.zeros((H, W))
    res = dict(filtered=out, A=A, new_mask=new_mask, valid=valid, vmin=None, vmax=None)
    if not valid.any():
        return res
    keys = f2key(depth[valid])
    vmin, vmax = key2f(keys.min()), key2f(keys.max())
    res.update(vmin=vmin, vmax=vmax)
    lo, rng = float(vmin), float(vmax) - float(vmin)
    with np.errstate(invalid="ignore", divide="ignore"):
        c = (depth.astype(np.float64) - lo) / rng
    c[~valid] = 0.0
    sc = float(f32(sigma_color))
    sc = 1.0 if sc <= 0 else sc
    gc = -0.5 / (sc * sc)
    ys, xs = reflect101(np.arange(-r, H + r), H), reflect101(np.arange(-r, W + r), W)
    pad = c[np.ix_(ys, xs)]
    # first-order error terms in units of u (module docstring):  nb = (dq - vmin) / rng_f has 3 roundings of nb
    dnb_c = 3 * c
    num, den = c.copy(), np.ones((H, W))
    s_abs, w_abs = c.copy(), np.ones((H, W))    # sum |terms| of the two window sums
    d_num, d_den = dnb_c.copy(), np.zeros((H, W))
    nterm = 1
    with np.errstate(invalid="ignore"):
        for dy, dx, ws in space_weights(r, sigma_space):
            nb = pad[r + dy:r + dy + H, r + dx:r + dx + W]
            diff = np.abs(nb - c)
            t = diff * diff * gc
            e = np.exp(t)
            w = ws * e
            ddiff = 3 * nb + dnb_c + diff
            dt = 2 * abs(gc) * diff * ddiff + 3 * np.abs(t)
            dw = ws * e * (dt + 4) + w
            num += nb * w
            den += w
            s_abs += nb * w
            w_abs += w
            d_num += w * 3 * nb + nb * dw + nb * w  # input errors and the product's rounding
            d_den += dw
            nterm += 1
        d_num += (nterm - 1) * s_abs
        d_den += (nterm - 1) * w_abs
        q = num / den
        dq = d_num / den + q * d_den / den + q
        filt = q * rng + lo
        A_v = rng * dq + 2 * q * rng + np.abs(filt)
    out[valid] = filt[valid]
    A[valid] = A_v[valid]
    return res


def flat_reflect101_old(i, n):
    """The border of the filter before OpenCV's repeated reflection: one reflection, out of the image when the
    radius reaches the image size."""
    i = np.asarray(i, np.int64)
    return np.where(i < 0, -i, np.where(i >= n, 2 * n - 2 - i, i))


def bilateral_with_reads(depth, mask, d, sigma_color, sigma_space, ymap, xmap):
    """bilateral64 where the window reads the flat element y * W + x of the arrays (clamped to the buffer), with
    (y, x) = (ymap(v + dy), xmap(u + dx)): what a kernel with that indexing reads from memory."""
    depth = np.asarray(depth, f32)
    H, W = depth.shape
    r = d // 2
    ref = bilateral64(depth, mask, d, sigma_color, sigma_space)
    if ref["vmin"] is None:
        return ref["filtered"]
    valid = ref["valid"]
    lo, rng = float(ref["vmin"]), float(ref["vmax"]) - float(ref["vmin"])
    with np.errstate(invalid="ignore", divide="ignore"):
        c = (depth.astype(np.float64) - lo) / rng
    c[~valid] = 0.0
    flat = c.reshape(-1)
    sc = float(f32(sigma_color))
    gc = -0.5 / (sc * sc)
    vv, uu = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    num, den = c.copy(), np.ones((H, W))
    for dy, dx, ws in space_weights(r, sigma_space):
        q = np.clip(ymap(vv + dy, H) * W + xmap(uu + dx, W), 0, H * W - 1)
        nb = flat[q]
        w = ws * np.exp((nb - c) ** 2 * gc)
        num += nb * w
        den += w
    out = ref["filtered"].copy()
    with np.errstate(invalid="ignore"):
        out[valid] = (num / den * rng + lo)[valid]
    return out


def check_bilateral(got_depth, got_mask, ref, depth, report=None, minmax=None):
    """The filter's outputs against bilateral64: new mask and min / max bit-exact, masked-out pixels restored bit for
    bit, every filtered pixel within EPS * A."""
    exact("bilateral: new_mask", np.asarray(got_mask, bool), ref["new_mask"])
    if minmax is not None:
        if ref["vmin"] is None:
            exact("bilateral: min/max", np.asarray(minmax, np.uint32), np.array([0xffffffff, 0], np.uint32))
        else:
            exact("bilateral: min/max", key2f(np.asarray(minmax, np.uint32)).view(np.uint32),
                  np.array([ref["vmin"], ref["vmax"]], f32).view(np.uint32))
    got = np.asarray(got_depth, f32)
    keep = ~ref["valid"]
    same_bits("bilateral: restored pixels", got[keep], np.asarray(depth, f32)[keep])
    return close("bilateral", got, ref["filtered"], ref["A"], report)


# ---- depth maps -----------------------------------------------------------------------------------------------------
def _pix(n):
    # Camera.depth2point's arange(n) / (n - 1) * (n - 1): the pixel index, NaN for n == 1 (0 / 0)
    return np.full(n, np.nan) if n == 1 else np.arange(n, dtype=np.float64)


def depth2point64(depth, fx, fy, cx, cy, c2w=None):
    """-> (points [H,W,3] f64, A [H,W,3]).  fx..cy as the C ABI takes them (float32)."""
    z = np.asarray(depth, f32).astype(np.float64)
    H, W = z.shape
    fx, fy, cx, cy = (float(f32(a)) for a in (fx, fy, cx, cy))
    u, v = _pix(W)[None, :], _pix(H)[:, None]
    with np.errstate(invalid="ignore"):
        T1x, T2x = u * z / fx, -cx * z / fx
        T1y, T2y = v * z / fy, -cy * z / fy
        x, y = (u - cx) * z / fx, (v - cy) * z / fy
        # u' = (u/(W-1))*(W-1) 2, u'*z 1, *ifx 1, ifx 1 | z*ox 1, ox 1 | the sum 1
        Ax = 5 * np.abs(T1x) + 2 * np.abs(T2x) + np.abs(x)
        Ay = 5 * np.abs(T1y) + 2 * np.abs(T2y) + np.abs(y)
    P = np.stack([x, y, z], -1)
    A = np.stack([Ax, Ay, np.zeros_like(z)], -1)
    if c2w is None:
        return P, A
    M = np.asarray(c2w, f32).astype(np.float64)
    with np.errstate(invalid="ignore"):
        Pw = P @ M[:3, :3].T + M[:3, 3]
        terms = np.abs(P) @ np.abs(M[:3, :3]).T + np.abs(M[:3, 3])
        Aw = A @ np.abs(M[:3, :3]).T + 3 * terms
    return Pw, Aw


def _ok(z, dmin, dmax):
    return (z > f32(dmin)) & (z < f32(dmax))   # float32 depths against the float32 thresholds: exact


def cross_normal64(depth, fx, fy, cx, cy, dmin=1e-3, dmax=100000.0):
    """-> (n [H,W,3] f64 camera normals, A [H,W,3], ok [H,W]) -- n and A are meaningful where ok."""
    z32 = np.asarray(depth, f32)
    H, W = z32.shape
    P, AP = depth2point64(z32, fx, fy, cx, cy)
    ok = np.zeros((H, W), bool)
    n = np.zeros((H, W, 3))
    A = np.zeros((H, W, 3))
    if H < 3 or W < 3:
        return n, A, ok
    okz = _ok(z32, dmin, dmax)
    ok[1:-1, 1:-1] = okz[1:-1, 1:-1] & okz[:-2, 1:-1] & okz[2:, 1:-1] & okz[1:-1, :-2] & okz[1:-1, 2:]
    sl = (slice(1, -1), slice(1, -1))
    with np.errstate(invalid="ignore", over="ignore"):
        a = P[:-2, 1:-1] - P[2:, 1:-1]
        h = P[1:-1, :-2] - P[1:-1, 2:]
        da = AP[:-2, 1:-1] + AP[2:, 1:-1] + np.abs(a)
        dh = AP[1:-1, :-2] + AP[1:-1, 2:] + np.abs(h)
        c = -np.cross(a, h)
        dc = np.zeros_like(c)
        for i, (j, k) in enumerate(((1, 2), (2, 0), (0, 1))):
            p1, p2 = a[..., j] * h[..., k], a[..., k] * h[..., j]
            dc[..., i] = (np.abs(h[..., k]) * da[..., j] + np.abs(a[..., j]) * dh[..., k] + np.abs(h[..., j]) * da[..., k]
                          + np.abs(a[..., k]) * dh[..., j] + np.abs(p1) + np.abs(p2) + np.abs(c[..., i]))
        ln = np.linalg.norm(c, axis=-1, keepdims=True)
        L = np.maximum(ln, 1e-12)
        nn = c / L
        dlen = (np.abs(c) * dc).sum(-1, keepdims=True) / L + 2.5 * ln
        dn = dc / L + np.abs(c) * dlen / L ** 2 + np.abs(nn)
    n[sl] = nn
    A[sl] = dn
    return n, A, ok


def depth2normal64(depth, fx, fy, cx, cy, dmin=1e-3, dmax=100000.0, rot=None):
    """ops.depth2normal: -> (n [H,W,3] f64 with the -1 fill, A [H,W,3], ok [H,W])."""
    n, A, ok = cross_normal64(depth, fx, fy, cx, cy, dmin, dmax)
    if rot is not None:
        n, A = rotate64(n, A, rot)
    n[~ok] = -1.0
    A[~ok] = 0.0
    return n, A, ok


def rotate64(n, A, rot):
    """n @ rot (row vectors) as the kernels evaluate it: three-term dot products."""
    R = np.asarray(rot, f32).astype(np.float64).reshape(3, 3)
    w = n @ R
    return w, A @ np.abs(R) + 3 * (np.abs(n) @ np.abs(R))


def fill_sum32(rot):
    """sum((-1, -1, -1) @ rot) as the kernel evaluates it in float32.  Every product is -rot_ij, exact, so the result
    does not depend on FMA contraction: w_j = (-r0j - r1j) - r2j, then (w0 + w1) + w2."""
    R = np.asarray(rot, f32).reshape(3, 3)
    w = [f32(f32(-R[0, j] - R[1, j]) - R[2, j]) for j in range(3)]
    return f32(f32(w[0] + w[1]) + w[2])


def view_normals64(filtered, fg, opacity, median_depth, fx, fy, cx, cy, rot, depth_limit, opacity_min=0.5):
    """extract_pcd.py:325-335 on the filtered depth and the dilated mask, as gsr_extract_normals computes it:
    -> dict(cam [H,W,3], A_cam, neg_world [H,W,3], A_world, valid [H,W], fill [H,W])."""
    n, A, ok = cross_normal64(filtered, fx, fy, cx, cy)
    fill = ~(ok & np.asarray(fg, bool))
    n[fill] = -1.0
    A[fill] = 0.0
    w, Aw = rotate64(n, A, rot)
    s32 = fill_sum32(rot)
    # the reference's literal rule; only the fill can come near -3 (|sum| <= sqrt(3) for a unit normal), and the
    # fill's sum is evaluated exactly above -- with an identity rotation it is -3 and the fill is never valid
    world_ok = np.where(fill, s32 > f32(-3.0), w.sum(-1) > -3.0)
    valid = world_ok & (np.asarray(median_depth, f32) < f32(depth_limit)) & (np.asarray(opacity, f32) > f32(opacity_min))
    return dict(cam=n, A_cam=A, neg_world=-w, A_world=Aw, valid=valid, fill=fill, ok=ok)


# ---- normal fusion --------------------------------------------------------------------------------------------------
def entry_weights64(xyz, cam_t, ids, normals, conf):
    """-> (w [m] f64, A_w [m]) for entries with ids in [0, P): conf * |dot(v/|v|, n)| / (|v| + 1e-6), v = t - xyz."""
    X = np.asarray(xyz, f32).astype(np.float64)[ids]
    t = np.asarray(cam_t, f32).astype(np.float64)
    n = np.asarray(normals, f32).astype(np.float64)
    c = np.asarray(conf, f32).astype(np.float64)
    v = t[None, :] - X
    dist = np.linalg.norm(v, axis=1)
    e = float(f32(1e-6))
    with np.errstate(invalid="ignore", divide="ignore"):
        vh = v / dist[:, None]
        dot = (vh * n).sum(1)
        w = c * np.abs(dot) / (dist + e)
        A = c / (dist + e) * 8 * np.abs(vh * n).sum(1) + 7 * w
    return w, A


def fusion_pass64(xyz, ids_list, normals_list, conf_list, cam_ts, mean=None, A_mean=None, thresh=0.8):
    """One pass: -> dict(sn [P,3], sw [P], A_sn, A_sw, touched [P], flagged [P] (a Gaussian with an entry whose
    consistency test lies within its bound of the threshold), n_flagged, margin (smallest |diff - thresh| / bound))."""
    P = np.asarray(xyz).shape[0]
    sn, sw = np.zeros((P, 3)), np.zeros(P)
    abs_sn, abs_sw, d_sn, d_sw = np.zeros((P, 3)), np.zeros(P), np.zeros((P, 3)), np.zeros(P)
    cnt = np.zeros(P)
    touched, flagged = np.zeros(P, bool), np.zeros(P, bool)
    margin = np.inf
    th = float(f32(thresh))
    for ids, nrm, conf, t in zip(ids_list, normals_list, conf_list, cam_ts):
        ids = np.asarray(ids, np.int64)
        keep = (ids >= 0) & (ids < P)
        ids = ids[keep]
        n = np.asarray(nrm, f32)[keep].astype(np.float64)
        w, Aw = entry_weights64(xyz, t, ids, n, np.asarray(conf, f32)[keep])
        touched[ids] = True
        if mean is not None:
            diff = np.linalg.norm(n - mean[ids], axis=1)
            with np.errstate(invalid="ignore"):
                bd = EPS * (A_mean[ids].sum(1) + 3 * diff)
                amb = np.abs(diff - th) <= bd
                if (~np.isnan(diff)).any():
                    margin = min(margin, float(np.nanmin(np.abs(diff - th) / np.maximum(bd, 1e-300))))
            flagged[ids[amb]] = True
            sel = diff < th
            ids, n, w, Aw = ids[sel], n[sel], w[sel], Aw[sel]
        nw = n * w[:, None]
        add = lambda x: np.bincount(ids, x, minlength=P)  # noqa: E731
        sw += add(w)
        abs_sw += add(np.abs(w))
        d_sw += add(Aw)
        cnt += add(np.ones(len(ids)))
        for i in range(3):
            sn[:, i] += add(nw[:, i])
            abs_sn[:, i] += add(np.abs(nw[:, i]))
            d_sn[:, i] += add(np.abs(n[:, i]) * Aw + np.abs(nw[:, i]))
    gain = np.maximum(cnt - 1, 0)
    A_sn = d_sn + gain[:, None] * abs_sn
    A_sw = d_sw + gain * abs_sw
    return dict(sn=sn, sw=sw, A_sn=A_sn, A_sw=A_sw, touched=touched, flagged=flagged, n_flagged=int(flagged.sum()),
                margin=margin)


def normalize64(x, Ax):
    """F.normalize(p=2, eps=1e-12) of rows x with input errors Ax -> (m, A_m)."""
    with np.errstate(invalid="ignore", divide="ignore"):
        ln = np.linalg.norm(x, axis=-1, keepdims=True)
        L = np.maximum(ln, 1e-12)
        m = x / L
        A = (Ax + np.abs(m) * (np.abs(m) * Ax).sum(-1, keepdims=True)) / L + 3.5 * np.abs(m)
    return m, A


def fusion_mean64(p):
    """k_fusion_mean: normalize(sum / weight), NaN where the weight is 0.  A sum that cancels exactly in float64 (terms
    that are exact negatives of each other) is asserted to be exactly 0 on the device too (check_mean), so its
    bound is 0 rather than the infinite conditioning of normalising a zero vector."""
    with np.errstate(invalid="ignore", divide="ignore"):
        x = p["sn"] / p["sw"][:, None]
        Ax = p["A_sn"] / p["sw"][:, None] + np.abs(x) * (p["A_sw"] / p["sw"])[:, None] + np.abs(x)
    m, A = normalize64(x, Ax)
    A[np.all(m == 0, axis=-1)] = 0.0
    return m, A


def fusion64(xyz, ids_list, normals_list, conf_list, cam_ts):
    """Both passes -> dict(p1, mean1, A1, p2, mean2, A2, uid)."""
    p1 = fusion_pass64(xyz, ids_list, normals_list, conf_list, cam_ts)
    m1, A1 = fusion_mean64(p1)
    p2 = fusion_pass64(xyz, ids_list, normals_list, conf_list, cam_ts, mean=m1, A_mean=A1)
    m2, A2 = fusion_mean64(p2)
    return dict(p1=p1, mean1=m1, A1=A1, p2=p2, mean2=m2, A2=A2, uid=np.nonzero(p1["touched"])[0])


def check_mean(check, got, m, A, skip=None, report=None):
    """A fusion mean: exactly 0 where the float64 sum cancels exactly, else within EPS * A; rows in `skip` (their
    pass-2 sums depend on a flagged decision) are not compared."""
    got = np.asarray(got, np.float64).copy()
    m = m.copy()
    zero = np.all(m == 0, axis=-1)
    exact(f"{check}: cancelled mean", got[zero], m[zero])
    if skip is not None:
        got[skip], m[skip] = 0.0, 0.0
    m[zero] = got[zero] = 0.0
    return close(check, got, m, A, report)


def smooth64(xyz_u, mean, A_mean, k=10, sigma=0.1):
    """normal_fusion's smoothing: normalize(sum_j mean[idx_j] * exp(-dist_j / 0.1)) over the exact k nearest points.
    -> (sm, A, ambiguous [n]: the k-th and (k+1)-th distances lie within the neighbour search's bound)."""
    n = len(xyz_u)
    k = min(k, n)
    sq, idx = knn64(xyz_u, k + 1 if n > k else k)
    d = np.sqrt(sq)
    amb = np.zeros(n, bool)
    if n > k:
        amb = d[:, k] - d[:, k - 1] <= 2 * knn_slack(xyz_u, d[:, k])
    d, idx = d[:, :k], idx[:, :k]
    e = np.exp(-d / sigma)
    with np.errstate(invalid="ignore"):
        s = (mean[idx] * e[..., None]).sum(1)
        # each neighbour's mean error, its distance's (4u relative) through the exp, the double sum's cast to float
        As = (A_mean[idx] * e[..., None] + np.abs(mean[idx]) * (e * 4 * d / sigma)[..., None]).sum(1) + np.abs(s)
    sm, A = normalize64(s, As)
    return sm, A, amb


# ---- k nearest neighbours -------------------------------------------------------------------------------------------
def knn64(pts, k, queries=None):
    """-> (squared distances [m, k] f64, indices [m, k]) of the float32 points, ordered by (distance, index)."""
    P = np.asarray(pts, f32).astype(np.float64)
    n = len(P)
    q = np.arange(n) if queries is None else np.asarray(queries)
    k = min(k, n)
    if n <= 6000:
        out_d, out_i = [], []
        for s in range(0, len(q), 512):
            Q = P[q[s:s + 512]]
            D = ((Q[:, None, :] - P[None, :, :]) ** 2).sum(-1)
            o = np.argsort(D, axis=1, kind="stable")[:, :k]
            out_d.append(np.take_along_axis(D, o, 1)); out_i.append(o)
        return np.concatenate(out_d), np.concatenate(out_i)
    from scipy.spatial import cKDTree
    kk = min(n, k + 8)
    _, cand = cKDTree(P).query(P[q], k=kk)
    D = ((P[q][:, None, :] - P[cand]) ** 2).sum(-1)
    o = np.lexsort((cand, D), axis=1)[:, :k]
    return np.take_along_axis(D, o, 1), np.take_along_axis(cand, o, 1)


def knn_slack(pts, d):
    """How far a distance may move by rounding in the grid search: 6u of the distance (the float32 squared distance
    and its sqrt) plus 4u of the box extent.  The cell of a point is floor((x - lo) * inv_h) in float32, so a cell
    boundary is only placed to within 2u |x - lo| for the query and for the point, and the stopping radius r * h can
    be short by that much."""
    P = np.asarray(pts, f32).astype(np.float64)
    ext = float((P.max(0) - P.min(0)).max()) if len(P) else 0.0
    return 6 * U * np.asarray(d) + 4 * U * ext


def check_knn(pts, got_dist, got_idx, k, queries=None, ref=None, report=None):
    """The neighbour search against knn64: indices unique and in range, each distance within 4u of the float64
    distance of the same index, ascending order, no point closer than the returned k-th one (beyond rounding) left
    out, and the returned k-th no farther than the true k-th (beyond rounding)."""
    P = np.asarray(pts, f32).astype(np.float64)
    n = len(P)
    q = np.arange(n) if queries is None else np.asarray(queries)
    gi = np.asarray(got_idx, np.int64)
    gd = np.asarray(got_dist, f32)
    k = min(k, n)
    if gi.shape != (len(q), k):
        fail("knn: indices", f"shape {gi.shape}, expected {(len(q), k)}")
    if (gi < 0).any() or (gi >= n).any():
        fail("knn: indices", "index out of range")
    srt = np.sort(gi, 1)
    if (srt[:, 1:] == srt[:, :-1]).any():
        fail("knn: indices", f"duplicate neighbour in {int((srt[:, 1:] == srt[:, :-1]).any(1).sum())} rows")
    sq = ((P[q][:, None, :] - P[gi]) ** 2).sum(-1)
    d64 = np.sqrt(sq)
    close("knn: distance", gd, d64, 2 * d64, report)      # EPS * 2d = 4u d
    if (np.diff(gd.astype(np.float64), axis=1) < 0).any():
        fail("knn: order", "returned distances are not ascending")
    if ref is None:
        ref = knn64(P.astype(f32), k, queries)
    rs, ri = ref
    true_k = np.sqrt(rs[:, k - 1])
    slack = knn_slack(P, np.maximum(true_k, d64[:, -1]))
    cut = d64[:, -1] - slack
    closer = np.sqrt(rs) < cut[:, None]
    present = (ri[:, :, None] == gi[:, None, :]).any(-1)
    missed = closer & ~present
    if missed.any():
        r = int(np.argwhere(missed.any(1))[0, 0])
        fail("knn: missed neighbour", f"{int(missed.any(1).sum())} rows leave out a point closer than their k-th, "
                                      f"first query {int(q[r])}")
    over = d64[:, -1] - true_k - slack
    if (over > 0).any():
        fail("knn: k-th cut", f"k-th distance exceeds the true k-th by {float(over.max()):.3e} beyond rounding")
    if report is not None:
        worst = float(np.max((d64[:, -1] - true_k) / np.maximum(slack, 1e-300))) if len(q) else 0.0
        report["knn: k-th cut"] = max(report.get("knn: k-th cut", -np.inf), worst)
