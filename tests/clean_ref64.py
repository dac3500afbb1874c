"""Float64 restatement of clean_point_cloud (gaustudio/scripts/extract_pcd.py:30-51), with the flagging rules that say
where the device may differ from it, and by how much.

Pass 1 restates Open3D's PointCloud::RemoveStatisticalOutliers: avg_i = mean of the min(k, N) nearest distances, the
point itself included; mean = sum avg / N; std = sqrt(sum_{avg > 0} (avg - mean)^2 / (N - 1)); keep avg > 0 and
avg < mean + r std.  Pass 2 restates remove_normal_outliers: the min(k2, N) - 1 nearest points other than i, the mean
of arccos(|n_i . n_j|) with |dot| clamped to 1 (or the reference's literal arccos), keep mean < theta.

Neighbours come from extract_ref64.knn64: squared distances (dx^2 + dy^2) + dz^2 in float64 of the float32 points,
ordered by (distance, index).

Flags (each check reports how many it found):
  pass-1 decisions with |avg_i - thr| within the rounding bound of avg_i plus that of thr (derived below);
  pass-2 decisions with |mean_i - theta| within the rounding bound of the mean angle;
  ties: points whose k2-th neighbour is at the same distance as the next one, where any choice among the tied points
        is an admissible neighbour set; the device must match the decision of one of them;
  duplicates: points with an exact copy, where the reference's idx[0] may be the copy rather than the point itself,
        so it drops the copy and keeps the point (angle 0); either choice is accepted.
"""
import numpy as np

from extract_ref64 import knn64

U64 = 2.0 ** -53
f32 = np.float32


def neighbours(xyz, k):
    """-> (sq [N, K], idx [N, K]) with K = min(k, N), the point itself among them: knn64, with its candidate search on
    every core for large clouds.  Candidates are the k + 8 nearest by the tree, re-ranked by the exact float64 key;
    clumps of more than k + 8 copies are ordered among themselves by index only in the small-cloud path."""
    P = np.asarray(xyz, f32)
    n = len(P)
    if n <= 6000:
        return knn64(P, k)
    from scipy.spatial import cKDTree
    k = min(k, n)
    P64 = P.astype(np.float64)
    _, cand = cKDTree(P64).query(P64, k=min(n, k + 8), workers=-1)
    out_d, out_i = [], []
    for s in range(0, n, 200_000):
        c = cand[s:s + 200_000]
        D = ((P64[s:s + 200_000, None, :] - P64[c]) ** 2).sum(-1)
        o = np.lexsort((c, D), axis=1)[:, :k]
        out_d.append(np.take_along_axis(D, o, 1)); out_i.append(np.take_along_axis(c, o, 1))
    return np.concatenate(out_d), np.concatenate(out_i)


# ---- pass 1 ----------------------------------------------------------------------------------------------------------
def statistical64(xyz, k=50, std_ratio=2.0, fault=None):
    """-> dict(avg, mean, std, thr, keep, bound_avg, bound_thr).  fault seeds one of the rule breaks the checks must
    catch: 'no_self' (self left out of the k), 'population' (std over N), 'le' (<= instead of <), 'no_pos' (avg > 0
    dropped)."""
    P = np.asarray(xyz, f32)
    N = len(P)
    if N == 0:
        e = np.zeros(0)
        return dict(avg=e, mean=np.nan, std=np.nan, thr=np.nan, keep=np.zeros(0, bool), bound_avg=e, bound_thr=0.0)
    if fault == "no_self":
        sq, idx = neighbours(P, min(k + 1, N))
        sq = sq[:, 1:] if N > 1 else sq
    else:
        sq, idx = neighbours(P, k)
    K = sq.shape[1]
    d = np.sqrt(sq)
    avg = d.sum(1) / K
    mean = avg[avg > 0].sum() / N
    dev2 = np.where(avg > 0, (avg - mean) ** 2, 0.0)
    with np.errstate(invalid="ignore", divide="ignore"):
        std = np.sqrt(dev2.sum() / (N if fault == "population" else N - 1))
    thr = mean + std_ratio * std
    below = avg <= thr if fault == "le" else avg < thr
    keep = below if fault == "no_pos" else (avg > 0) & below
    # Rounding bounds, in units of the double unit roundoff u.  The device forms the same squared distances and
    # correctly rounded square roots, and sums the K distances in another order: (K - 1) u sum d on each side, u for
    # the division.  mean: N u of the sum of avg on each side, plus the mean of the avg bounds.  The squared
    # deviations move by 2 |avg - mean| (b_avg + b_mean) each, their sums by N u each; std = sqrt(s / (N - 1)) moves
    # by b_s / (2 (N - 1) std) + u std; thr by b_mean + r b_std + 2 u thr.
    b_avg = (2.0 * (K - 1) + 2.0) * U64 * avg
    b_mean = b_avg.mean() + 2.0 * N * U64 * mean
    s = dev2.sum()
    b_s = (2.0 * np.abs(avg - mean) * (b_avg + b_mean))[avg > 0].sum() + 2.0 * N * U64 * s
    with np.errstate(invalid="ignore", divide="ignore"):
        b_std = b_s / (2.0 * (N - 1) * std) + 2.0 * U64 * std if std > 0 else np.sqrt(b_s / max(N - 1, 1))
    b_thr = b_mean + std_ratio * b_std + 2.0 * U64 * abs(thr)
    return dict(avg=avg, mean=mean, std=std, thr=thr, keep=keep, bound_avg=b_avg, bound_thr=b_thr, K=K)


def flag_statistical(ref):
    """Decisions within rounding of the threshold."""
    with np.errstate(invalid="ignore"):
        return np.abs(ref["avg"] - ref["thr"]) < ref["bound_avg"] + ref["bound_thr"]


# ---- pass 2 ----------------------------------------------------------------------------------------------------------
def angles(n_i, n_j, literal=False):
    dot = (n_j.astype(np.float64) * n_i.astype(np.float64)).sum(-1)
    x = np.abs(dot)
    if not literal:
        x = np.where(x > 1.0, 1.0, x)  # NaN stays NaN
    with np.errstate(invalid="ignore"):
        return np.arccos(x)


def normal64(xyz, normals, k=20, theta=np.pi / 4, literal=False, fault=None):
    """-> dict(mean, keep, bound, tie, dup, lo, hi).  literal: the reference's arccos without the clamp.  fault:
    'idx0' (idx[0] not excluded: the point itself counted, the last neighbour left out), 'over_k' (divide by k instead of k - 1),
    'fmin' (clamp with fmin, which turns NaN into 1)."""
    P = np.asarray(xyz, f32)
    Nr = np.asarray(normals, f32)
    N = len(P)
    if N == 0:
        e = np.zeros(0)
        return dict(mean=e, keep=np.zeros(0, bool), bound=e, tie=np.zeros(0, bool), dup=np.zeros(0, bool), lo=e, hi=e)
    K = min(k, N)
    extra = min(K + 1, N)
    sq, idx = neighbours(P, extra)
    me = np.arange(N)
    # the K - 1 nearest points other than i, in (distance, index) order
    if fault == "idx0":
        pick = np.broadcast_to(np.arange(K - 1), (N, K - 1))
    else:
        pick = np.argsort(idx == me[:, None], axis=1, kind="stable")[:, :K - 1]
    others, osq = np.take_along_axis(idx, pick, 1), np.take_along_axis(sq, pick, 1)
    m = K - 1
    if m > 0:
        a = angles(Nr[:, None, :], Nr[others], literal)
        if fault == "fmin":
            dot = np.abs((Nr[others].astype(np.float64) * Nr[:, None, :].astype(np.float64)).sum(-1))
            a = np.arccos(np.fmin(dot, 1.0))
        with np.errstate(invalid="ignore"):
            mean = a.sum(1) / (k if fault == "over_k" else m)
    else:
        a = np.zeros((N, 0))
        mean = np.full(N, np.nan)
    with np.errstate(invalid="ignore"):
        keep = mean < theta
    # bound: the same dot products; acos within 2 ulp on the device (<= 4 u |a|) and 1 ulp here; the sum in another
    # order, (m - 1) u sum a on each side; the division u
    with np.errstate(invalid="ignore"):
        bound = ((2.0 * max(m - 1, 0) + 6.0) * U64 * np.abs(a).sum(1) / max(m, 1) + 2.0 * U64 * np.abs(mean))
    # ties at the cut: the K-th nearest (self included) at the distance of the (K+1)-th
    tie = np.zeros(N, bool)
    lo, hi = mean.copy(), mean.copy()
    if extra > K and m > 0:
        tie = sq[:, K - 1] == sq[:, K]
        for r in np.nonzero(tie)[0]:
            dcut = sq[r, K - 1]
            D = ((P[r].astype(np.float64) - P.astype(np.float64)) ** 2).sum(-1)
            pool = np.nonzero((D == dcut) & (me != r))[0]
            fixed = others[r][osq[r] < dcut]
            t = m - len(fixed)
            af = angles(Nr[r], Nr[fixed], literal)
            ap = np.sort(angles(Nr[r], Nr[pool], literal))  # NaN last
            lo[r] = (af.sum() + ap[:t].sum()) / m
            hi[r] = (af.sum() + ap[-t:].sum()) / m
    # exact copies: the reference may drop a copy instead of the point itself and keep the point's own angle 0
    dup = np.zeros(N, bool)
    if N > 1:
        dup = sq[:, 1] == 0
    return dict(mean=mean, keep=keep, bound=bound, tie=tie, dup=dup, lo=lo, hi=hi, others=others, osq=osq, angles=a, m=m)


def dup_variants(ref, normals, r, theta, literal=False):
    """Decisions of point r when the reference drops one of its exact copies instead of itself (self's angle counted)."""
    Nr = np.asarray(normals, f32)
    a, m = ref["angles"][r], ref["m"]
    self_angle = angles(Nr[r], Nr[r][None], literal)[0]
    out = set()
    for j in np.nonzero(ref["osq"][r] == 0)[0]:
        b = np.concatenate([np.delete(a, j), [self_angle]])
        with np.errstate(invalid="ignore"):
            out.add(bool(b.sum() / m < theta))
    return out


def flag_normal(ref, theta=np.pi / 4):
    with np.errstate(invalid="ignore"):
        return np.abs(ref["mean"] - theta) < ref["bound"]


class CheckError(AssertionError):
    pass


def check_statistical(avg, keep, ref, report=None):
    """Device avg within bound per element; decisions equal except flagged ones.  -> number flagged."""
    avg = np.asarray(avg, np.float64)
    keep = np.asarray(keep, bool)
    err = np.abs(avg - ref["avg"])
    bad = err > ref["bound_avg"]
    if bad.any():
        i = int(np.argmax(bad))
        raise CheckError(f"pass 1: avg off by {err[i]:.3e} > bound {ref['bound_avg'][i]:.3e} at {i}")
    flag = flag_statistical(ref)
    wrong = (keep != ref["keep"]) & ~flag
    if wrong.any():
        raise CheckError(f"pass 1: {int(wrong.sum())} decisions differ from float64, first {int(np.argmax(wrong))}")
    if report is not None:
        ratio = float((err / np.maximum(ref["bound_avg"], 1e-300)).max()) if len(err) else 0.0
        report["pass1 flagged"] = report.get("pass1 flagged", 0) + int(flag.sum())
        report["pass1 worst err/bound"] = max(report.get("pass1 worst err/bound", 0.0), ratio)
    return int(flag.sum())


def check_normal(mean, keep, ref, normals, theta=np.pi / 4, report=None):
    """Device mean angles within bound (NaN where float64 is NaN), decisions equal except flagged ones, and flagged
    ties / duplicates consistent with an admissible neighbour set.  -> dict of flag counts."""
    mean = np.asarray(mean, np.float64)
    keep = np.asarray(keep, bool)
    want = ref["mean"]
    if not np.array_equal(np.isnan(mean), np.isnan(want)):
        raise CheckError(f"pass 2: NaN pattern differs at {int((np.isnan(mean) != np.isnan(want)).sum())} points")
    fin = ~np.isnan(want)
    err = np.abs(mean[fin] - want[fin])
    bad = err > ref["bound"][fin]
    if bad.any():
        raise CheckError(f"pass 2: mean angle off by {err.max():.3e} beyond its bound")
    near = flag_normal(ref, theta)
    wrong = (keep != ref["keep"]) & ~near
    if wrong.any():
        raise CheckError(f"pass 2: {int(wrong.sum())} decisions differ from float64, first {int(np.argmax(wrong))}")
    # ties: keep possible iff the lowest admissible mean is < theta, drop possible iff the highest is >= theta or NaN
    for r in np.nonzero(ref["tie"])[0]:
        ok_keep = ref["lo"][r] < theta
        ok_drop = not (ref["hi"][r] < theta)
        if (keep[r] and not ok_keep) or (not keep[r] and not ok_drop):
            raise CheckError(f"pass 2: point {r} (tied cut) matches no admissible neighbour set")
    for r in np.nonzero(ref["dup"])[0]:
        allowed = {bool(ref["keep"][r])} | dup_variants(ref, normals, r, theta)
        if bool(keep[r]) not in allowed and not near[r]:
            raise CheckError(f"pass 2: point {r} (exact copy) matches neither choice of the excluded point")
    counts = {"near theta": int(near.sum()), "ties": int(ref["tie"].sum()), "duplicates": int(ref["dup"].sum())}
    if report is not None:
        for c, v in counts.items():
            report[f"pass2 {c}"] = report.get(f"pass2 {c}", 0) + v
        ratio = float((err / np.maximum(ref["bound"][fin], 1e-300)).max()) if err.size else 0.0
        report["pass2 worst err/bound"] = max(report.get("pass2 worst err/bound", 0.0), ratio)
    return counts


def clean64(xyz, normals, k=50, std_ratio=2.0, k2=20, theta=np.pi / 4, literal=False):
    """Both passes -> (index, ref1, ref2, first)."""
    r1 = statistical64(xyz, k, std_ratio)
    first = np.nonzero(r1["keep"])[0]
    r2 = normal64(np.asarray(xyz)[first], np.asarray(normals)[first], k2, theta, literal)
    return first[r2["keep"]], r1, r2, first


# ---- scenes ----------------------------------------------------------------------------------------------------------
def surface(kind, n, seed=0):
    """(xyz, normals) float32 on a unit-size sphere, plane or torus."""
    g = np.random.default_rng(seed)
    if kind == "sphere":
        d = g.normal(size=(n, 3))
        nr = d / np.linalg.norm(d, axis=1, keepdims=True)
        p = 0.5 * nr
    elif kind == "plane":
        p = np.c_[g.uniform(-0.5, 0.5, (n, 2)), np.zeros(n)]
        nr = np.tile([0.0, 0.0, 1.0], (n, 1))
    else:
        u, v = g.uniform(0, 2 * np.pi, (2, n))
        R, r = 0.4, 0.15
        c = np.c_[np.cos(u), np.sin(u), np.zeros(n)]
        nr = c * np.cos(v)[:, None] + np.c_[np.zeros((n, 2)), np.sin(v)]
        p = R * c + r * nr
    return p.astype(f32), nr.astype(f32)


def with_floaters(xyz, normals, frac, far=1.0, seed=1):
    """Adds round(frac * N) floaters uniform in a box `far` times the scene's size, with random unit normals."""
    g = np.random.default_rng(seed)
    m = int(round(frac * len(xyz)))
    f = g.uniform(-0.5, 0.5, (m, 3)) * 2.0 * far
    fn = g.normal(size=(m, 3))
    fn /= np.linalg.norm(fn, axis=1, keepdims=True)
    return np.r_[xyz, f.astype(f32)], np.r_[normals, fn.astype(f32)], np.arange(len(xyz), len(xyz) + m)
