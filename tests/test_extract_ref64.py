"""The float64 restatements of the extraction kernels (tests/extract_ref64.py) against the reference's outputs, the
numpy oracle, OpenCV and independent formulas; and every checker of tests/test_gpu_extract_f64.py fed a seeded fault,
each of which must be reported by its own check."""
import os

import numpy as np
import pytest

import extract_ref64 as R
from oracle import extract_oracle as eo

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "extract_golden.npz"))
f32 = np.float32

TINY = [(1, 7, 3), (7, 1, 3), (2, 5, 5), (3, 3, 7), (2, 2, 5), (1, 3, 15), (1, 1, 3), (4, 9, 15), (5, 7, 15)]


def _golden_bilateral(case):
    kw = {}
    if case == "s":
        kw = dict(sigma_color=float(G["bil_s_sigma"][0]), sigma_space=float(G["bil_s_sigma"][1]))
    return G[f"bil_{case}_depth"], G[f"bil_{case}_mask"], int(G[f"bil_{case}_d"]), kw


@pytest.mark.parametrize("case", ["a", "b", "c", "s"])
def test_bilateral64_matches_reference_and_oracle(case):
    depth, mask, d, kw = _golden_bilateral(case)
    ref = R.bilateral64(depth, mask, d, **kw)
    assert np.array_equal(ref["new_mask"], G[f"bil_{case}_newmask"].astype(bool))
    # OpenCV's 4096-bin range table against the direct exp, on a ~2 unit depth range
    np.testing.assert_allclose(ref["filtered"], G[f"bil_{case}_filtered"], rtol=0, atol=2e-6)
    fo, mo = eo.masked_bilateral_filter(depth, mask, d, **kw)   # a float32 evaluation: inside the kernel's bound
    assert np.array_equal(mo, ref["new_mask"])
    assert R.check_bilateral(fo, mo, ref, depth) < 0.5


def _cv2_masked_bilateral(cv2, depth, mask, d, sc, ss):
    """extract_pcd.py's masked_bilateral_filter, restated on cv2.dilate / cv2.bilateralFilter."""
    dil = cv2.dilate((~mask).astype(np.uint8), np.ones((d, d), np.uint8))
    new_mask = dil == 0
    valid = new_mask & ~np.isnan(depth)
    out = depth.copy()
    if valid.any():
        lo, hi = depth[valid].min(), depth[valid].max()
        with np.errstate(invalid="ignore", divide="ignore"):
            nd = (depth - lo) / (hi - lo)
        nd[~valid] = 0
        f = cv2.bilateralFilter(nd.astype(np.float32), d=d, sigmaColor=sc, sigmaSpace=ss)
        out = f * (hi - lo) + lo
        out[~valid] = depth[~valid]
    return out, new_mask


@pytest.mark.parametrize("H,W,d", TINY)
def test_bilateral64_matches_opencv_on_images_smaller_than_the_window(H, W, d):
    """OpenCV reflects again until the index is inside (and uses 0 when the side is 1 pixel)."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(H * 100 + W * 10 + d)
    depth = (1 + rng.random((H, W))).astype(f32)
    for mask in (np.ones((H, W), bool), rng.random((H, W)) > 0.2):
        ref = R.bilateral64(depth, mask, d, 0.3, 2.0)
        co, cm = _cv2_masked_bilateral(cv2, depth, mask, d, 0.3, 2.0)
        assert np.array_equal(cm, ref["new_mask"])
        if ref["valid"].sum() == 1:   # a zero depth range: 0 / 0 in the reference as well
            assert np.isnan(ref["filtered"][ref["valid"]]).all() and np.isnan(co[ref["valid"]]).all()
            continue
        np.testing.assert_allclose(ref["filtered"], co, rtol=0, atol=2e-6)


@pytest.mark.parametrize("H,W,d", TINY)
def test_oracle_filters_images_smaller_than_the_window(H, W, d):
    depth = (1 + np.random.default_rng(d).random((H, W))).astype(f32)
    mask = np.ones((H, W), bool)
    fo, mo = eo.masked_bilateral_filter(depth, mask, d, 0.3, 2.0)
    ref = R.bilateral64(depth, mask, d, 0.3, 2.0)
    if ref["valid"].sum() == 1:
        assert np.isnan(fo).all() and np.isnan(ref["filtered"]).all()
    else:
        assert R.check_bilateral(fo, mo, ref, depth) < 0.5


def test_minmax_keys_order_signed_zeros_and_negatives():
    x = np.array([0.0, -0.0, -3.5, 2.0, np.inf, -np.inf], f32)
    k = R.f2key(x)
    assert np.array_equal(R.key2f(k).view(np.uint32), x.view(np.uint32))
    assert list(np.argsort(k)) == [5, 2, 1, 0, 3, 4]
    depth = np.array([[0.0, -0.0, 1.0]], f32)
    ref = R.bilateral64(depth, np.ones((1, 3), bool), 1)
    assert ref["vmin"].view(np.uint32) == f32(-0.0).view(np.uint32) and ref["vmax"] == 1


def _plane_depth(n, c, H, W, fx, fy, cx, cy):
    """Depth of the plane n . X = c seen through pixel (u, v): z = c / (n . ((u - cx)/fx, (v - cy)/fy, 1))."""
    u, v = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    ray = np.stack([(u - cx) / fx, (v - cy) / fy, np.ones_like(u)], -1)
    return c / (ray @ n), ray


@pytest.mark.parametrize("n", [(0, 0, 1), (0.3, -0.2, 1), (0.9, 0.1, 0.3), (-0.2, 0.9, 0.35)])
def test_cross_normal_against_a_plane_fit(n):
    """On a plane the 5-point cross normal is the plane's normal, oriented along the viewing ray."""
    n = np.asarray(n, np.float64) / np.linalg.norm(n)
    H, W, fx, fy, cx, cy = 24, 31, 120.0, 124.0, 13.0, 10.5
    z, ray = _plane_depth(n, 3.0, H, W, fx, fy, cx, cy)
    z32 = z.astype(f32)
    got, A, ok = R.cross_normal64(z32, fx, fy, cx, cy)
    assert ok[1:-1, 1:-1].all() and not ok[0].any() and not ok[:, -1].any()
    P, _ = R.depth2point64(z32, fx, fy, cx, cy)
    for (v, u) in [(5, 7), (12, 15), (H - 2, W - 2)]:
        nb = np.stack([P[v, u], P[v - 1, u], P[v + 1, u], P[v, u - 1], P[v, u + 1]])
        fit = np.linalg.svd(nb - nb.mean(0))[2][-1]          # least-squares plane through the five points
        fit *= np.sign(fit @ ray[v, u])
        np.testing.assert_allclose(got[v, u], fit, atol=1e-6)
        np.testing.assert_allclose(got[v, u], n * np.sign(n @ ray[v, u]), atol=1e-5)


def test_depth2normal64_matches_oracle_and_camera_golden():
    C = np.load(os.path.join(os.path.dirname(__file__), "golden", "camera_golden.npz"))
    for i in range(4):
        K = C[f"c{i}_K"]
        d = C[f"c{i}_depth"]
        n, A, ok = R.depth2normal64(d, K[0, 0], K[1, 1], K[0, 2], K[1, 2])
        assert R.close("depth2normal", C[f"c{i}_normal_cam"], n, A) < 1
        ext = C[f"c{i}_view"].T
        rot = np.linalg.inv(ext[:3, :3].astype(np.float64)).T.astype(f32)
        nw, Aw, _ = R.depth2normal64(d, K[0, 0], K[1, 1], K[0, 2], K[1, 2], rot=rot)
        assert R.close("depth2normal", C[f"c{i}_normal_world"], nw, Aw) < 1
        p, Ap = R.depth2point64(d, K[0, 0], K[1, 1], K[0, 2], K[1, 2])
        assert R.close("depth2point", C[f"c{i}_point_cam"], p, Ap) < 1


def test_view_normals64_matches_oracle_and_pins_the_fill_rule():
    """sum(fill @ rot) > -3 only recognises the (-1, -1, -1) fill under the identity rotation: with a rotated camera
    the fill pixels pass it and are valid when their median depth and opacity pass (the reference's behaviour)."""
    rng = np.random.default_rng(3)
    H, W = 30, 40
    depth = (2 + 0.05 * rng.random((H, W))).astype(f32)
    depth[5:9, 5:12] = 0       # invalid depths: filled
    fg = rng.random((H, W)) > 0.1
    op = rng.random((H, W)).astype(f32)
    md = (2 + rng.random((H, W))).astype(f32)
    th = 0.4
    E = np.eye(4, dtype=f32)
    E[:3, :3] = np.array([[np.cos(th), 0, np.sin(th)], [0, 1, 0], [-np.sin(th), 0, np.cos(th)]], f32)
    for ext, fill_valid in ((np.eye(4, dtype=f32), False), (E, True)):
        rot = np.linalg.inv(ext[:3, :3]).T.astype(f32)
        o = eo.view_normals(depth, fg, op, md, np.zeros((H, W), np.int32), 30.0, 31.0, 19.5, 14.5, ext, 3.5)
        r = R.view_normals64(depth, fg, op, md, 30.0, 31.0, 19.5, 14.5, rot, f32(3.5 * 0.8))
        assert np.array_equal(r["valid"], o["valid"])
        assert R.close("extract_normals: camera", o["cam_normals"], r["cam"], r["A_cam"]) < 1
        assert bool((r["valid"] & r["fill"]).any()) == fill_valid


def _fusion_golden():
    V = int(G["fus_V"])
    return (G["fus_xyz"], [G[f"fus_ids{v}"] for v in range(V)], [G[f"fus_n{v}"] for v in range(V)],
            [G[f"fus_c{v}"] for v in range(V)], [G[f"fus_E{v}"][:3, 3] for v in range(V)])


def test_fusion64_matches_reference_and_oracle():
    xyz, ids, nrm, conf, ts = _fusion_golden()
    f = R.fusion64(xyz, ids, nrm, conf, ts)
    assert np.array_equal(f["uid"], G["fus_unique_ids"])
    assert f["p2"]["n_flagged"] == 0
    ouid, omean = eo.normal_fusion(xyz, ids, nrm, conf, ts, smooth=False)
    assert R.check_mean("fusion: mean", omean, f["mean2"][f["uid"]], f["A2"][f["uid"]]) < 1
    sm, A, amb = R.smooth64(np.asarray(xyz, f32)[f["uid"]], f["mean2"][f["uid"]], f["A2"][f["uid"]])
    ref = G["fus_smoothed"]
    assert np.array_equal(np.isnan(sm), np.isnan(ref)) and not amb.any()
    np.testing.assert_allclose(np.nan_to_num(sm), np.nan_to_num(ref), rtol=0, atol=2e-6)


def test_knn64_matches_ckdtree():
    from scipy.spatial import cKDTree
    p = np.random.default_rng(1).standard_normal((7000, 3)).astype(f32)
    for q in (None, np.arange(0, 7000, 7)):
        sq, idx = R.knn64(p, 10, q)
        d, i = cKDTree(p.astype(np.float64)).query(p[np.arange(7000) if q is None else q].astype(np.float64), k=10)
        assert np.array_equal(idx, i)
        np.testing.assert_allclose(np.sqrt(sq), d, rtol=1e-12)
    sq, idx = R.knn64(p[:3000], 10)   # brute force path
    d, i = cKDTree(p[:3000].astype(np.float64)).query(p[:3000].astype(np.float64), k=10)
    assert np.array_equal(idx, i)
    sq, idx = R.knn64(np.zeros((20, 3), f32), 4)  # ties by index
    assert (idx == np.arange(4)).all()


# ---- seeded faults: each one must be caught, by its own check ----------------------------------------------------
def _fires(check, fn):
    with pytest.raises(R.CheckError) as e:
        fn()
    assert str(e.value).startswith(check + ":"), str(e.value)


def test_fault_border_reflected_once_is_caught_by_the_bilateral_check():
    """The single reflection the filter used before reads outside the image once the radius reaches its size."""
    rng = np.random.default_rng(7)
    for H, W, d in [(1, 7, 3), (4, 2, 5), (3, 6, 15)]:
        depth = (1 + rng.random((H, W))).astype(f32)
        mask = np.ones((H, W), bool)
        ref = R.bilateral64(depth, mask, d, 0.3, 2.0)
        R.check_bilateral(ref["filtered"].astype(f32), ref["new_mask"], ref, depth)   # the clean result passes
        bad = R.bilateral_with_reads(depth, mask, d, 0.3, 2.0, R.flat_reflect101_old, R.flat_reflect101_old)
        _fires("bilateral", lambda: R.check_bilateral(bad.astype(f32), ref["new_mask"], ref, depth))
        good = R.bilateral_with_reads(depth, mask, d, 0.3, 2.0, R.reflect101, R.reflect101)
        R.check_bilateral(good.astype(f32), ref["new_mask"], ref, depth)


def _knn_case(k=10):
    p = np.random.default_rng(2).random((400, 3)).astype(f32)
    sq, idx = R.knn64(p, k + 1)
    return p, sq, idx


def test_fault_neighbour_replaced_by_the_next_one_is_caught_by_the_missed_neighbour_check():
    p, sq, idx = _knn_case()
    R.check_knn(p, np.sqrt(sq[:, :10]).astype(f32), idx[:, :10], 10)
    gi, gd = idx[:, :10].copy(), np.sqrt(sq[:, :10]).astype(f32)
    gi[17, 9], gd[17, 9] = idx[17, 10], f32(np.sqrt(sq[17, 10]))
    _fires("knn: missed neighbour", lambda: R.check_knn(p, gd, gi, 10))


def test_knn_checker_reports_duplicates_distances_and_order():
    p, sq, idx = _knn_case()
    gi, gd = idx[:, :10].copy(), np.sqrt(sq[:, :10]).astype(f32)
    g2 = gi.copy(); g2[3, 4] = g2[3, 5]
    _fires("knn: indices", lambda: R.check_knn(p, gd, g2, 10))
    d2 = gd.copy(); d2[3, 4] = np.nextafter(np.nextafter(d2[3, 4], f32(9)), f32(9)) * f32(1 + 2 ** -20)
    _fires("knn: distance", lambda: R.check_knn(p, d2, gi, 10))
    g3, d3 = gi.copy(), gd.copy()
    g3[3, [4, 5]], d3[3, [4, 5]] = g3[3, [5, 4]], d3[3, [5, 4]]
    _fires("knn: order", lambda: R.check_knn(p, d3, g3, 10))


def _fusion_case():
    rng = np.random.default_rng(11)
    P, V, m = 60, 4, 150
    xyz = rng.standard_normal((P, 3)).astype(f32)
    ts = [rng.standard_normal(3).astype(f32) * 6 for _ in range(V)]
    ids = [rng.integers(0, P, m) for _ in range(V)]
    base = rng.standard_normal((P, 3))
    base /= np.linalg.norm(base, axis=1, keepdims=True)
    nrm = []
    for i in ids:
        n = base[i] + 0.2 * rng.standard_normal((m, 3))
        nrm.append((n / np.linalg.norm(n, axis=1, keepdims=True)).astype(f32))
    conf = [rng.random(m).astype(f32) for _ in range(V)]
    return xyz, ids, nrm, conf, ts


def test_fault_dropped_fusion_term_is_caught_by_the_fusion_sum_check():
    xyz, ids, nrm, conf, ts = _fusion_case()
    f = R.fusion64(xyz, ids, nrm, conf, ts)
    p = f["p1"]
    R.close("fusion: sums", p["sn"].astype(f32), p["sn"], p["A_sn"])
    keep = np.ones(len(ids[1]), bool); keep[5] = False
    ids2 = [ids[0], ids[1][keep]] + ids[2:]
    nrm2 = [nrm[0], nrm[1][keep]] + nrm[2:]
    conf2 = [conf[0], conf[1][keep]] + conf[2:]
    bad = R.fusion_pass64(xyz, ids2, nrm2, conf2, ts)
    _fires("fusion: sums", lambda: R.close("fusion: sums", bad["sn"].astype(f32), p["sn"], p["A_sn"]))


def test_fault_flipped_normal_is_caught_by_the_normal_check():
    rng = np.random.default_rng(5)
    depth = (3 + 0.2 * rng.random((20, 26))).astype(f32)
    n, A, ok = R.depth2normal64(depth, 25.0, 25.0, 12.0, 9.0)
    got = n.astype(f32)
    R.close("depth2normal", got, n, A)
    got[7, 9] *= -1
    _fires("depth2normal", lambda: R.close("depth2normal", got, n, A))


def test_fault_point_off_by_64_ulp_is_caught_by_the_point_check():
    rng = np.random.default_rng(6)
    H, W = 12, 17
    depth = (2 + rng.random((H, W))).astype(f32)
    p, A = R.depth2point64(depth, 20.0, 21.0, 8.3, 5.7)
    got = p.astype(f32)
    R.close("depth2point", got, p, A)
    v, u = 4, W - 1
    uz_ifx = abs(f32(f32(u) * depth[v, u]) * (f32(1) / f32(20.0)))
    got[v, u, 0] += 64 * np.spacing(f32(uz_ifx))
    _fires("depth2point", lambda: R.close("depth2point", got, p, A))
