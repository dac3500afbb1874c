"""-m gpu: the extraction kernels against their float64 contracts (tests/extract_ref64.py), element by element, with
no outlier budget.

  gsr_masked_bilateral   k_dilate_minmax + k_bilateral: images smaller than the window, every d, masks that touch
                         each border, NaN / negative / signed-zero depths, depth ranges from 1e-6 to 1e4, 1920x1080
  gsr_depth2point        k_depth2point, camera and world coordinates (a c2w with a 1e3 translation)
  gsr_depth2normal       k_depth2normal: depths at dmin / dmax and one ulp either side, NaN / 0 / inf, off-centre
                         principal points, grazing planes, rotations
  gsr_extract_normals    k_extract_normals through extract_view on a rendered 1920x1080 orbit view
  gsr_normal_fusion_*    k_fusion_pass / k_fusion_mean: both passes, the strict < 0.8, opposing normals, a camera on a
                         Gaussian, ids -1 and >= P; then normal_fusion's smoothing
  gsr_knn_grid           k_knn_grid for k in {1, 4, 8, 10, 16}: n = k + 1, lattices on cell edges, 1000 copies of one
                         point, far clusters, a plane, a line, a 1e4 offset, 2.2 M points

The worst |gpu - ref| / bound of every check and the flagged counts are printed at the end of the module (-s).
"""
import math

import numpy as np
import pytest
import torch

import extract_ref64 as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
f32 = np.float32
REPORT = {}
FLAGGED = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\n[extract f64] worst |gpu - ref| / bound:")
    for k in sorted(REPORT):
        print(f"  {k:32s} {REPORT[k]:.3f}")
    print("[extract f64] flagged:", dict(sorted(FLAGGED.items())))


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _poison():
    """Leave NaN in the memory the caching allocator hands out next, so outputs the kernels fail to write show."""
    t = torch.full((64 << 20,), float("nan"), device=DEV)
    del t


# ---- masked bilateral filter ----------------------------------------------------------------------------------------
def _bilateral_raw(depth, mask, d, sc, ss):
    """gsr_masked_bilateral with NaN-filled outputs, a mask output of 0xAA and the min / max words read back."""
    from gaustudio_b200._lib import call, ptr
    H, W = depth.shape
    dg, mg = cu(depth), cu(mask.astype(np.uint8))
    out = torch.full((H, W), float("nan"), device=DEV)
    nm = torch.full((H, W), 0xAA, dtype=torch.uint8, device=DEV)
    scratch = torch.full((2,), 0x5A5A5A5A, dtype=torch.int32, device=DEV)
    call("gsr_masked_bilateral", dg.device, ptr(dg), ptr(mg), W, H, d, float(sc), float(ss), ptr(out), ptr(nm), ptr(scratch))
    nm = nm.cpu().numpy()
    assert np.isin(nm, (0, 1)).all(), "new_mask: an element was not written"
    return out.cpu().numpy(), nm.astype(bool), scratch.cpu().numpy().view(np.uint32)


def _masks(H, W, rng):
    ys, xs = np.mgrid[:H, :W]
    holes = np.ones((H, W), bool)
    holes[0, W // 2] = holes[H - 1, (W - 1) // 3] = holes[H // 2, 0] = holes[(H - 1) // 3, W - 1] = False
    one = np.zeros((H, W), bool)
    one[H // 2, W // 2] = True
    return {"all": np.ones((H, W), bool), "none": np.zeros((H, W), bool), "checker": (ys + xs) % 2 == 0,
            "border_holes": holes, "random": rng.random((H, W)) > 0.1, "one": one}


def _depths(H, W, rng):
    base = rng.random((H, W))
    signed = (2 * base - 1).astype(f32)
    flat = signed.reshape(-1)
    flat[::7] = np.nan
    flat[3::11] = -0.0
    flat[5::13] = 0.0
    return {"plain": (1 + base).astype(f32), "nan_neg_zero": signed, "range_1e-6": (1 + 1e-6 * base).astype(f32),
            "range_1e4": (1e4 * base).astype(f32)}


SIZES = [(1, 1), (1, 37), (37, 1), (2, 2), (3, 3), (7, 5), (33, 9)]


@pytest.mark.parametrize("H,W", SIZES)
def test_bilateral_small_images_every_window_and_mask(H, W):
    rng = np.random.default_rng(H * 1000 + W)
    for d in (1, 3, 5, 7, 15):
        for mname, mask in _masks(H, W, rng).items():
            for dname, depth in _depths(H, W, rng).items():
                for sc, ss in ((75.0, 75.0), (0.2, 2.0)):
                    ref = R.bilateral64(depth, mask, d, sc, ss)
                    got, nm, mm = _bilateral_raw(depth, mask, d, sc, ss)
                    try:
                        R.check_bilateral(got, nm, ref, depth, REPORT, minmax=mm)
                    except R.CheckError as e:
                        raise AssertionError(f"{H}x{W} d={d} mask={mname} depth={dname} sigma={sc},{ss}: {e}")


@pytest.mark.parametrize("d", [3, 15])
def test_bilateral_full_size(d):
    rng = np.random.default_rng(d)
    H, W = 1080, 1920
    depth = (2 + 3 * rng.random((H, W))).astype(f32)
    depth[400:420, 900:1300] = np.nan
    mask = rng.random((H, W)) > 0.02
    mask[:, :3] = False
    mask[-2:, :] = False
    ref = R.bilateral64(depth, mask, d, 0.3, 4.0)
    got, nm, mm = _bilateral_raw(depth, mask, d, 0.3, 4.0)
    R.check_bilateral(got, nm, ref, depth, REPORT, minmax=mm)
    # the Python entry gives the same bits
    from gaustudio_b200.extract import masked_bilateral_filter
    f, m = masked_bilateral_filter(cu(depth), cu(mask), d=d, sigma_color=0.3, sigma_space=4.0)
    R.same_bits("bilateral: python entry", f.cpu().numpy(), got)
    R.exact("bilateral: python entry", m.cpu().numpy(), nm)


# ---- depth maps ------------------------------------------------------------------------------------------------------
def _depth_map(H, W, rng, kind, fx, fy, cx, cy):
    u, v = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    if kind == "grazing":   # a plane seen nearly edge-on: z grows fast along u, the cross product cancels
        n = np.array([0.995, 0.05, 0.0866])
        ray = np.stack([(u - cx) / fx, (v - cy) / fy, np.ones_like(u)], -1)
        z = 2.0 / np.abs(ray @ n)
    else:
        z = 2 + 0.5 * np.sin(u / 5.0) + 0.3 * np.cos(v / 3.0) + 0.05 * rng.random((H, W))
    z = z.astype(f32)
    if kind == "edges":
        dmin, dmax = f32(1e-3), f32(1e5)
        vals = [dmin, np.nextafter(dmin, f32(0)), np.nextafter(dmin, f32(1)), dmax, np.nextafter(dmax, f32(0)),
                np.nextafter(dmax, f32(np.inf)), f32(np.nan), f32(0), f32(np.inf), f32(-1)]
        flat = z.reshape(-1)
        idx = rng.choice(flat.size, min(flat.size, 4 * len(vals)), replace=False)
        flat[idx] = np.resize(np.array(vals, f32), len(idx))
    return z


def _rot(a, b):
    ca, sa, cb, sb = math.cos(a), math.sin(a), math.cos(b), math.sin(b)
    Rz = np.array([[ca, -sa, 0], [sa, ca, 0], [0, 0, 1]])
    Rx = np.array([[1, 0, 0], [0, cb, -sb], [0, sb, cb]])
    return (Rz @ Rx).astype(f32)


@pytest.mark.parametrize("H,W", SIZES + [(1080, 1920)])
def test_depth2point_and_depth2normal(H, W):
    from gaustudio_b200 import ops
    rng = np.random.default_rng(H + 7 * W)
    for kind in ("smooth", "grazing", "edges"):
        for fx, fy, cx, cy in ((0.9 * W + 3, 0.9 * W + 3, W / 2, H / 2), (1.3 * W + 5, 1.1 * W + 5, 0.17 * W, 0.81 * H)):
            depth = _depth_map(H, W, rng, kind, fx, fy, cx, cy)
            dg = cu(depth)
            fin = np.isfinite(depth)
            c2w = np.eye(4, dtype=f32)
            c2w[:3, :3] = _rot(0.7, -0.4)
            c2w[:3, 3] = (1e3, -2.5e2, 7e2)
            for M in (None, c2w):
                _poison()
                got = ops.depth2point(dg, fx, fy, cx, cy, cam_to_world=None if M is None else cu(M)).cpu().numpy()
                ref, A = R.depth2point64(depth, fx, fy, cx, cy, M)
                # non-finite depths give non-finite points (the reference's 0 * inf and inf - inf)
                assert not np.isfinite(got[~fin]).all(axis=-1).any()
                if M is None:
                    R.same_bits("depth2point: z", got[..., 2], depth)
                R.close("depth2point" if M is None else "depth2point: world", got[fin], ref[fin], A[fin], REPORT)
            for rot in (None, _rot(0.3, 1.1)):
                _poison()
                got = ops.depth2normal(dg, fx, fy, cx, cy, rot=None if rot is None else cu(rot)).cpu().numpy()
                ref, A, ok = R.depth2normal64(depth, fx, fy, cx, cy, rot=rot)
                R.exact("depth2normal: fill", np.all(got == -1, axis=-1) & ~ok, ~ok)
                R.close("depth2normal" if rot is None else "depth2normal: rotated", got, ref, A, REPORT)


# ---- one rendered view, extract_view(compact=False) through to normal_fusion --------------------------------------
def _views(H, W, K, P):
    from gaustudio_b200 import extract, renderers
    from gaustudio_b200.synthetic import build_config
    model, cams, _ = build_config("cfg1", P=P, W=W, H=H, K=K)
    model.to(torch.device(DEV))
    cams = [c.to(torch.device(DEV)) for c in cams]
    r = renderers.make({"name": "vanilla_renderer"})
    radius = extract.getNerfppNorm(cams)["radius"]
    out = []
    for cam in cams:
        with torch.no_grad():
            pkg = r.render(cam, model)
        _poison()
        v = extract.extract_view(cam, pkg, radius, compact=False)
        out.append((cam, pkg, v))
    return model, cams, radius, out


def _check_view(cam, pkg, v, radius):
    from gaustudio_b200 import extract
    depth = pkg["rendered_depth"][0].cpu().numpy()
    op = pkg["rendered_final_opacity"][0].cpu().numpy()
    md = pkg["rendered_median_depth"][0].cpu().numpy()
    mi = pkg["rendered_median_id"][0].cpu().numpy()
    ref = R.bilateral64(depth, op > f32(0.1), 3, 75.0, 75.0)
    filt, fg = v["filtered_depth"].cpu().numpy(), v["fg_mask"].cpu().numpy()
    R.check_bilateral(filt, fg, ref, depth, REPORT)
    fx, fy, cx, cy = extract._intrinsics_host(cam)
    rot = np.linalg.inv(extract._extrinsics_host(cam)[:3, :3]).T.astype(f32)
    assert abs(float(np.trace(rot)) - 3) > 1e-3   # a rotated camera: the fill is not recognised, as in the reference
    o = R.view_normals64(filt, fg, op, md, fx, fy, cx, cy, rot, f32(radius * 0.8))
    R.close("extract_normals: camera", v["cam_normals"].cpu().numpy(), o["cam"], o["A_cam"], REPORT)
    valid = v["valid"].cpu().numpy()
    R.exact("extract_normals: valid", valid, o["valid"])
    R.close("extract_normals: world", v["normals"].cpu().numpy().reshape(o["neg_world"].shape), o["neg_world"],
            o["A_world"], REPORT)
    R.exact("extract_normals: ids", v["ids"].cpu().numpy(), np.where(o["valid"], mi, -1).reshape(-1))
    R.same_bits("extract_normals: confidences", v["confidences"].cpu().numpy(), op.reshape(-1))
    return (o["valid"] & o["fill"]).sum(), o["valid"].sum()


def _gpu_fusion(xyz, ids, nrm, conf, ts):
    """normal_fusion's two passes through the C entries, keeping each pass's sums and means."""
    from gaustudio_b200 import extract
    X = cu(np.asarray(xyz, f32))
    P = X.shape[0]
    sums, weights = torch.zeros(P, 3, device=DEV), torch.zeros(P, device=DEV)
    touched = torch.zeros(P, dtype=torch.uint8, device=DEV)
    ids = [torch.as_tensor(i).to(DEV) for i in ids]
    nrm = [torch.as_tensor(n).to(DEV) for n in nrm]
    conf = [torch.as_tensor(c).to(DEV) for c in conf]
    ts = [[float(a) for a in t] for t in ts]
    m1 = extract._fusion_pass(X, ids, nrm, conf, ts, None, sums, weights, touched)
    s1, w1 = sums.cpu().numpy(), weights.cpu().numpy()
    sums.zero_(); weights.zero_()
    m2 = extract._fusion_pass(X, ids, nrm, conf, ts, m1, sums, weights, None)
    return dict(s1=s1, w1=w1, m1=m1.cpu().numpy(), s2=sums.cpu().numpy(), w2=weights.cpu().numpy(),
                m2=m2.cpu().numpy(), touched=touched.cpu().numpy().astype(bool))


def _check_fusion(xyz, ids, nrm, conf, ts, name, max_flagged=0):
    ref = R.fusion64(xyz, ids, nrm, conf, ts)
    g = _gpu_fusion(xyz, ids, nrm, conf, ts)
    R.exact(f"{name}: touched", g["touched"], ref["p1"]["touched"])
    p1, p2 = ref["p1"], ref["p2"]
    R.close(f"{name}: pass 1 sums", g["s1"], p1["sn"], p1["A_sn"], REPORT)
    R.close(f"{name}: pass 1 weights", g["w1"], p1["sw"], p1["A_sw"], REPORT)
    R.check_mean(f"{name}: pass 1 mean", g["m1"], ref["mean1"], ref["A1"], report=REPORT)
    fl = p2["flagged"]
    FLAGGED[name] = FLAGGED.get(name, 0) + int(fl.sum())
    assert fl.sum() <= max_flagged, f"{name}: {int(fl.sum())} Gaussians with an entry within its bound of 0.8"
    keep = ~fl
    R.close(f"{name}: pass 2 sums", g["s2"][keep], p2["sn"][keep], p2["A_sn"][keep], REPORT)
    R.close(f"{name}: pass 2 weights", g["w2"][keep], p2["sw"][keep], p2["A_sw"][keep], REPORT)
    R.check_mean(f"{name}: mean", g["m2"], ref["mean2"], ref["A2"], skip=fl, report=REPORT)
    return ref, fl


def _check_smoothing(xyz, ids, nrm, conf, cams, ref, fl, name):
    from gaustudio_b200 import extract
    uid, sm = extract.normal_fusion(type("PC", (), {"_xyz": cu(np.asarray(xyz, f32))})(), ids, nrm, conf, cams)
    R.exact(f"{name}: unique ids", uid.cpu().numpy(), ref["uid"])
    u = ref["uid"]
    s64, A, amb = R.smooth64(np.asarray(xyz, f32)[u], ref["mean2"][u], ref["A2"][u])
    # rows whose neighbour set is not decided by rounding, or that take a flagged Gaussian's mean
    _, nb = R.knn64(np.asarray(xyz, f32)[u], min(10, len(u)))
    near_flagged = fl[u][nb].any(1)
    skip = amb | near_flagged
    FLAGGED[f"{name}: ambiguous neighbour sets"] = FLAGGED.get(f"{name}: ambiguous neighbour sets", 0) + int(amb.sum())
    FLAGGED[f"{name}: rows reading a flagged mean"] = (FLAGGED.get(f"{name}: rows reading a flagged mean", 0)
                                                      + int((near_flagged & ~amb).sum()))
    assert amb.sum() <= 1 + 1e-3 * len(u)
    got = sm.cpu().numpy().astype(np.float64)
    got[skip], s64[skip] = 0.0, 0.0
    R.close(f"{name}: smoothed", got, s64, A, REPORT)


def test_extract_view_to_normal_fusion_full_size_rotated_cameras():
    model, cams, radius, views = _views(1080, 1920, 3, 100_000)
    xyz = model._xyz.detach().cpu().numpy()
    ids, nrm, conf, ts = [], [], [], []
    for cam, pkg, v in views:
        nfill, nvalid = _check_view(cam, pkg, v, radius)
        FLAGGED["view: valid fill pixels"] = FLAGGED.get("view: valid fill pixels", 0) + int(nfill)
        assert nvalid > 1000
        ids.append(v["ids"].cpu().numpy()); nrm.append(v["normals"].cpu().numpy())
        conf.append(v["confidences"].cpu().numpy())
        from gaustudio_b200 import extract
        ts.append(extract._extrinsics_host(cam)[:3, 3])
    n_entries = sum(int((i >= 0).sum()) for i in ids)
    ref, fl = _check_fusion(xyz, ids, nrm, conf, ts, "fusion: rendered", max_flagged=max(1, n_entries // 10000))
    _check_smoothing(xyz, [torch.as_tensor(i) for i in ids], [torch.as_tensor(n) for n in nrm],
                     [torch.as_tensor(c) for c in conf], cams, ref, fl, "fusion: rendered")


def _fusion_scene(seed, P=3000, V=6, m=4000):
    rng = np.random.default_rng(seed)
    xyz = rng.standard_normal((P, 3)).astype(f32)
    ts = [(rng.standard_normal(3) * 5).astype(f32) for _ in range(V)]
    base = rng.standard_normal((P, 3))
    base /= np.linalg.norm(base, axis=1, keepdims=True)
    ids, nrm, conf = [], [], []
    for _ in range(V):
        i = rng.integers(0, P - 10, m)
        n = base[i] + 0.15 * rng.standard_normal((m, 3))
        flip = rng.random(m) < 0.03              # outliers far beyond 0.8 from the mean
        n[flip] *= -1
        ids.append(i); nrm.append((n / np.linalg.norm(n, axis=1, keepdims=True)).astype(f32))
        conf.append(rng.random(m).astype(f32))
    # ids outside [0, P): skipped
    ids[0] = np.concatenate([ids[0], [-1, P, P + 5, -7]])
    nrm[0] = np.concatenate([nrm[0], np.ones((4, 3), f32)])
    conf[0] = np.concatenate([conf[0], np.ones(4, f32)])
    # Gaussian P-1: observed twice with opposing normals and equal weights, so the mean cancels exactly
    g = P - 1
    ids[1] = np.concatenate([ids[1], [g, g]])
    nrm[1] = np.concatenate([nrm[1], np.array([[0.6, 0, 0.8], [-0.6, 0, -0.8]], f32)])
    conf[1] = np.concatenate([conf[1], np.full(2, 0.7, f32)])
    # Gaussian P-2 sits on camera 2 (dist = 0): NaN weight, NaN mean, as in the reference
    xyz[P - 2] = ts[2]
    ids[2] = np.concatenate([ids[2], [P - 2]])
    nrm[2] = np.concatenate([nrm[2], np.array([[0, 0, 1]], f32)])
    conf[2] = np.concatenate([conf[2], np.ones(1, f32)])
    return xyz, ids, nrm, conf, ts


@pytest.mark.parametrize("seed", [0, 1])
def test_fusion_passes(seed):
    xyz, ids, nrm, conf, ts = _fusion_scene(seed)
    ref, fl = _check_fusion(xyz, ids, nrm, conf, ts, "fusion")
    P = len(xyz)
    assert np.all(ref["mean2"][P - 1] == 0) or np.isnan(ref["mean2"][P - 1]).all()
    assert np.isnan(ref["mean2"][P - 2]).all() and np.all(ref["mean1"][P - 1] == 0)
    assert ref["p2"]["margin"] > 1, "an entry lies within its bound of 0.8"
    cams = [type("C", (), {"extrinsics": torch.from_numpy(np.block([[np.eye(3, dtype=f32), t[:, None]],
                                                                     [np.zeros((1, 3), f32), np.ones((1, 1), f32)]]))})()
            for t in ts]
    _check_smoothing(xyz, [torch.as_tensor(i) for i in ids], [torch.as_tensor(n) for n in nrm],
                     [torch.as_tensor(c) for c in conf], cams, ref, fl, "fusion")


def test_fusion_consistency_test_is_strict():
    """|n - mean| against 0.8f: entries at one ulp below 0.8f count, entries at 0.8f and one ulp above do not."""
    from gaustudio_b200._lib import call, ptr
    th = f32(0.8)
    xs = [np.nextafter(th, f32(0)), th, np.nextafter(th, f32(1)), f32(0.5), f32(0.9)]
    P = len(xs)
    n = np.zeros((P, 3), f32)
    n[:, 0] = xs
    for x in xs:   # |(x, 0, 0) - 0| is x exactly in float32 and in float64
        assert np.sqrt(f32(x * x)) == x
    ids = cu(np.arange(P, dtype=np.int64))
    xyz = cu(np.zeros((P, 3), f32))
    mean = cu(np.zeros((P, 3), f32))
    sums, weights = torch.zeros(P, 3, device=DEV), torch.zeros(P, device=DEV)
    ng, cg = cu(n), cu(np.ones(P, f32))
    call("gsr_normal_fusion_pass", ids.device, P, ptr(ids), ptr(ng), ptr(cg), P, ptr(xyz), 3.0, 0.0, 0.0, ptr(mean), 0.8,
         ptr(sums), ptr(weights), None)
    w = weights.cpu().numpy()
    ref = np.array([x < th for x in xs])
    R.exact("fusion: strict < 0.8", w > 0, ref)
    wr, Aw = R.entry_weights64(np.zeros((P, 3), f32), f32([3, 0, 0]), np.arange(P), n, np.ones(P, f32))
    R.close("fusion: entry weight", w[ref], wr[ref], Aw[ref], REPORT)


# ---- k nearest neighbours --------------------------------------------------------------------------------------------
def _knn_points(case, k):
    rng = np.random.default_rng(k)
    if case == "k+1":
        return rng.random((k + 1, 3)).astype(f32)
    if case == "lattice":   # power-of-two spacing: every point on a cell edge of knn's grid as well
        g = np.arange(12, dtype=f32) * f32(0.25)
        return np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    if case == "copies":
        return np.tile(np.array([[0.3, -1.2, 2.5]], f32), (1000, 1))
    if case == "clusters":
        a = rng.standard_normal((800, 3)) * 0.01
        b = rng.standard_normal((200, 3)) * 0.01 + 1e3
        return np.concatenate([a, b]).astype(f32)
    if case == "plane":
        p = rng.random((5000, 3))
        p[:, 2] = 0.25
        return p.astype(f32)
    if case == "line":
        p = np.zeros((3000, 3))
        p[:, 0] = rng.random(3000)
        return p.astype(f32)
    if case == "offset_1e4":
        return (rng.random((5000, 3)) + 1e4).astype(f32)
    if case == "shell":
        p = rng.standard_normal((40000, 3))
        return (p / np.linalg.norm(p, axis=1, keepdims=True)).astype(f32)
    raise KeyError(case)


KS = (1, 4, 8, 10, 16)


@pytest.mark.parametrize("case", ["k+1", "lattice", "copies", "clusters", "plane", "line", "offset_1e4", "shell"])
def test_knn_against_float64(case):
    from gaustudio_b200.extract import knn
    for k in KS:
        p = _knn_points(case, k)
        _poison()
        dist, idx = knn(cu(p), k=k)
        try:
            R.check_knn(p, dist.cpu().numpy(), idx.cpu().numpy(), k, report=REPORT)
        except R.CheckError as e:
            raise AssertionError(f"{case} k={k}: {e}")
        if case == "copies":   # every distance 0: ties go to the lower index
            assert (idx.cpu().numpy() == np.arange(k)).all() and float(dist.abs().max()) == 0


def _knn_raw(p, k, lo, inv_h, dims):
    """gsr_knn_grid on a grid given by the caller (the cells of an exact power-of-two width)."""
    from gaustudio_b200._lib import call, ptr
    cell = np.minimum(np.maximum(np.floor((p - lo) * inv_h), 0), np.array(dims) - 1).astype(np.int64)
    cid = (cell[:, 2] * dims[1] + cell[:, 1]) * dims[0] + cell[:, 0]
    order = np.argsort(cid, kind="stable")
    start = np.concatenate([[0], np.cumsum(np.bincount(cid, minlength=int(np.prod(dims))))]).astype(np.int32)
    grid = np.array([*lo, inv_h, *dims, 0], f32)
    sp, cs, gr = cu(p[order]), cu(start), cu(grid)
    oi = torch.full((len(p), k), -7, dtype=torch.int32, device=DEV)
    od = torch.full((len(p), k), float("nan"), device=DEV)
    call("gsr_knn_grid", sp.device, len(p), k, ptr(sp), ptr(cs), ptr(gr), ptr(oi), ptr(od))
    idx = np.empty((len(p), k), np.int64)
    dist = np.empty((len(p), k), f32)
    idx[order] = order[oi.cpu().numpy()]
    dist[order] = od.cpu().numpy()
    return dist, idx


@pytest.mark.parametrize("inv_h", [4.0, 2.0, 1.0])
def test_knn_points_exactly_on_cell_edges(inv_h):
    """Lattice spacing 0.25 and a cell width of 0.25, 0.5 or 1: (x - lo) * inv_h is an exact integer for every
    point, so each point sits on the lower edge of its cell, and the stopping radius r * h is met with equality."""
    g = np.arange(10, dtype=f32) * f32(0.25)
    p = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    dims = [int(np.floor(2.25 * inv_h)) + 1] * 3
    for k in KS:
        dist, idx = _knn_raw(p, k, np.zeros(3, f32), inv_h, dims)
        try:
            R.check_knn(p, dist, idx, k, report=REPORT)
        except R.CheckError as e:
            raise AssertionError(f"inv_h={inv_h} k={k}: {e}")


def test_knn_large_cloud_grid_clamped():
    """2.2 M points: the grid clamps at 256 cells a side; 20 000 sampled queries against cKDTree in float64."""
    from gaustudio_b200.extract import knn
    rng = np.random.default_rng(22)
    n = 2_200_000
    p = rng.standard_normal((n, 3))
    p = (p / np.linalg.norm(p, axis=1, keepdims=True) * (1 + 0.02 * rng.standard_normal((n, 1)))).astype(f32)
    q = rng.choice(n, 20000, replace=False)
    pg = cu(p)
    for k in KS:
        dist, idx = knn(pg, k=k)
        ref = R.knn64(p, k, q)
        R.check_knn(p, dist.cpu().numpy()[q], idx.cpu().numpy()[q], k, queries=q, ref=ref, report=REPORT)
