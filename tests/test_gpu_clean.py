"""-m gpu: point-cloud cleaning on the device (extract.remove_statistical_outlier / remove_normal_outliers /
clean_point_cloud, csrc/gsr_clean.cu) against the float64 restatement of tests/clean_ref64.py, with no outlier budget:
every decision and returned index equals float64's except flagged elements, the per-point mean distances and mean
angles lie within their bounds, the neighbour search meets check_knn, results repeat bit for bit and do not depend on
what the allocator's blocks held, and extract_pcd -> clean_point_cloud -> mesh_sap removes rendered floaters."""
import math

import numpy as np
import pytest
import torch

import clean_ref64 as C
import extract_ref64 as R
from gaustudio_b200 import _lib, extract

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
REPORT = {}


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(DEV)


def device_stat(xyz, k, ratio=2.0):
    n = len(xyz)
    avg = torch.empty(n, dtype=torch.float64, device=DEV)
    stats = torch.empty(3, dtype=torch.float64, device=DEV)
    keep = torch.empty(n, dtype=torch.uint8, device=DEV)
    with _lib.scratch(DEV):
        _lib.call("gsr_clean_statistical", DEV, n, _lib.ptr(xyz), k, float(ratio), _lib.ALLOC, 1, _lib.ptr(avg),
                  _lib.ptr(stats), _lib.ptr(keep))
    return avg.cpu().numpy(), keep.cpu().numpy().astype(bool), stats.cpu().numpy()


def device_angle(xyz, normals, k, theta=math.pi / 4):
    n = len(xyz)
    mean = torch.empty(n, dtype=torch.float64, device=DEV)
    keep = torch.empty(n, dtype=torch.uint8, device=DEV)
    with _lib.scratch(DEV):
        _lib.call("gsr_clean_normal", DEV, n, _lib.ptr(xyz), _lib.ptr(normals), k, float(theta), _lib.ALLOC, 1,
                  _lib.ptr(mean), _lib.ptr(keep))
    return mean.cpu().numpy(), keep.cpu().numpy().astype(bool)


def device_knn(xyz, k):
    n = len(xyz)
    idx = torch.full((n, k), -1, dtype=torch.int32, device=DEV)
    d2 = torch.empty(n, k, dtype=torch.float64, device=DEV)
    with _lib.scratch(DEV):
        _lib.call("gsr_clean_knn", DEV, n, _lib.ptr(xyz), k, _lib.ALLOC, 1, _lib.ptr(idx), _lib.ptr(d2))
    K = min(k, n)
    return idx.cpu().numpy()[:, :K], d2.cpu().numpy()[:, :K]


def scene(kind, n, frac=0.0, far=1.0, seed=0):
    x, nr = C.surface(kind, n, seed)
    if frac:
        x, nr, _ = C.with_floaters(x, nr, frac, far, seed + 1)
    return x, nr


def check_both(x, nr, k=50, ratio=2.0, k2=20):
    """Pass 1 on x, pass 2 on its float64 survivors, through the device entries and the public functions."""
    xd = cu(x)
    avg, keep, stats = device_stat(xd, k, ratio)
    r1 = C.statistical64(x, k, ratio)
    C.check_statistical(avg, keep, r1, REPORT)
    got1 = extract.remove_statistical_outlier(xd, k, ratio).cpu().numpy()
    assert np.array_equal(got1, np.nonzero(keep)[0])
    first = np.nonzero(r1["keep"])[0]
    if len(first) == 0:
        return
    xs, ns = x[first], nr[first]
    mean, keep2 = device_angle(cu(xs), cu(ns), k2)
    r2 = C.normal64(xs, ns, k2)
    C.check_normal(mean, keep2, r2, ns, report=REPORT)
    got2 = extract.remove_normal_outliers(cu(xs), cu(ns), k2).cpu().numpy()
    assert np.array_equal(got2, np.nonzero(keep2)[0])


@pytest.mark.parametrize("N", [1, 2, 3, 17, 64, 65, 1000])
def test_small_clouds(N):
    x, nr = scene("sphere", N, seed=N)
    check_both(x, nr)


@pytest.mark.parametrize("k", [1, 2, 20, 49, 50, 64])
def test_k_against_float64(k):
    x, nr = scene("torus", 20_000, 0.01, 2.0, seed=k)
    check_both(x, nr, k=k, k2=max(k, 2))


@pytest.mark.parametrize("kind,frac,far", [("sphere", 0.001, 1.0), ("plane", 0.01, 3.0), ("torus", 0.05, 1.5),
                                           ("sphere", 0.01, 1000.0), ("torus", 0.02, 1000.0)])
def test_surfaces_with_floaters(kind, frac, far):
    x, nr = scene(kind, 200_000, frac, far, seed=3)
    check_both(x, nr)
    print(kind, frac, far, REPORT)


def test_million_point_sphere_with_five_percent_far_floaters():
    """Floaters alone in their cells are 5 % of the cloud: the search must still start at the surface's density."""
    x, nr = scene("sphere", 1_000_000, 0.05, 1000.0, seed=3)
    check_both(x, nr)


def test_two_million_points_pass1():
    x, _ = scene("sphere", 2_000_000, 0.01, 1000.0, seed=9)
    avg, keep, _ = device_stat(cu(x), 50)
    C.check_statistical(avg, keep, C.statistical64(x, 50), REPORT)


def test_duplicates_and_clumps():
    x, nr = scene("plane", 20_000, seed=4)
    g = np.random.default_rng(4)
    x = np.r_[x, x[:500], np.tile(x[600:601], (80, 1)), np.tile(np.float32([[0.2, 0.1, 0.3]]), (70, 1))]
    nr = np.r_[nr, g.normal(size=(500, 3)).astype(np.float32), np.tile(nr[600:601], (80, 1)),
               np.tile(np.float32([[0, 1, 0]]), (70, 1))]
    check_both(x, nr)


def test_nan_normals_are_dropped_with_their_neighbourhoods():
    x, nr = scene("sphere", 50_000, seed=5)
    nr[::97] = np.nan
    check_both(x, nr)
    _, _, _, index = extract.clean_point_cloud(cu(x), cu(nr), cu(nr))
    assert not np.isin(np.arange(0, len(x), 97), index.cpu().numpy()).any()


def test_236_plane_is_kept_whole():
    nv = torch.nn.functional.normalize(torch.tensor([[2.0, 3.0, 6.0]]), dim=1).numpy()[0]
    g = np.random.default_rng(2).uniform(-1, 1, (30_000, 2))
    e1 = np.cross(nv, [1.0, 0, 0]); e1 /= np.linalg.norm(e1)
    e2 = np.cross(nv, e1)
    x = (g[:, :1] * e1 + g[:, 1:] * e2).astype(np.float32)
    n = np.tile(nv, (len(x), 1)).astype(np.float32)
    got = extract.remove_normal_outliers(cu(x), cu(n)).cpu().numpy()
    assert len(got) == len(x)
    check_both(x, n)


@pytest.mark.parametrize("k", [50, 64])
def test_knn_contract(k):
    x, _ = scene("torus", 100_000, 0.02, 1000.0, seed=k)
    idx, d2 = device_knn(cu(x), k)
    sq, ri = C.neighbours(x, k)
    assert np.array_equal(d2, sq)  # the same float64 squared distances, in the same order
    q = np.arange(0, len(x), 7)
    R.check_knn(x, np.sqrt(d2[q]).astype(np.float32), idx[q], k, queries=q, ref=(sq[q], ri[q]), report=REPORT)
    small = np.random.default_rng(k).normal(size=(3000, 3)).astype(np.float32)
    idx, d2 = device_knn(cu(small), k)
    sq, ri = R.knn64(small, k)
    assert np.array_equal(idx, ri) and np.array_equal(d2, sq)


def test_same_bits_on_two_runs_and_after_junk_in_the_allocator():
    x, nr = scene("sphere", 300_000, 0.01, 1000.0, seed=11)
    xd, nd = cu(x), cu(nr)
    a = device_stat(xd, 50), device_angle(xd, nd, 20)
    torch.cuda.empty_cache()
    junk = [torch.full((k,), float("nan"), device=DEV) for k in (1 << 10, 1 << 16, 1 << 20, 1 << 22, 1 << 24, 1 << 25)]
    junk += [torch.full((1 << 22,), -7, dtype=torch.int32, device=DEV) for _ in range(4)]
    del junk  # the caching allocator keeps these blocks and hands them out again
    b = device_stat(xd, 50), device_angle(xd, nd, 20)
    for u, v in ((a[0][0], b[0][0]), (a[0][1], b[0][1]), (a[0][2], b[0][2]), (a[1][0], b[1][0]), (a[1][1], b[1][1])):
        assert np.array_equal(u.view(np.uint8), v.view(np.uint8))
    c1 = extract.clean_point_cloud(xd, nd, nd)
    c2 = extract.clean_point_cloud(xd, nd, nd)
    assert all(torch.equal(p, q) for p, q in zip(c1, c2))


def test_device_refusals():
    x = torch.rand(10, 3, device=DEV)
    x[3, 1] = float("nan")
    with pytest.raises(ValueError, match="finite"):
        extract.remove_statistical_outlier(x)
    assert extract.remove_statistical_outlier(torch.empty(0, 3, device=DEV)).numel() == 0


def test_extract_pcd_clean_then_mesh_sap_removes_rendered_floaters():
    """The sphere of test_gpu_sap's extract_pcd -> mesh_sap test, plus opaque floater Gaussians outside it: every
    floater's fused point is removed, the decisions match float64, and the mesh of the cleaned cloud stays within 2 %
    of R with no NaN-row filtering by the caller."""
    from gaustudio_b200 import renderers
    from gaustudio_b200.camera import orbit_cameras
    from gaustudio_b200.synthetic import GaussianPointCloud
    R0, P, F = 0.6, 60_000, 40
    g = torch.Generator().manual_seed(7)
    d = torch.randn(P, 3, generator=g)
    d = d / d.norm(dim=1, keepdim=True)
    fd = torch.randn(F, 3, generator=g)
    fd = fd / fd.norm(dim=1, keepdim=True) * (R0 * (1.25 + 0.5 * torch.rand(F, 1, generator=g)))
    xyz0 = torch.cat([R0 * d, fd])
    pcd = GaussianPointCloud(xyz0, torch.full((P + F, 3), math.log(0.012)), torch.randn(P + F, 4, generator=g),
                             torch.full((P + F, 1), 4.0), torch.randn(P + F, 1, 3, generator=g),
                             torch.zeros(P + F, 15, 3), 3, 0)
    pcd.to(DEV)
    fov = math.radians(40.0)
    cams = orbit_cameras(16, 2.5, 35.0, 160, 160, fov, fov) + orbit_cameras(16, 2.5, -35.0, 160, 160, fov, fov)
    cams = [c.to(DEV) for c in cams]
    xyz, rgb, normals, _ = extract.extract_pcd(renderers.make({"name": "vanilla_renderer"}), pcd, cams)
    xyz = xyz.detach().float().contiguous()
    normals, rgb = normals.float().contiguous(), rgb.float().contiguous()
    x_np, n_np = xyz.cpu().numpy(), normals.cpu().numpy()
    floater = np.linalg.norm(x_np.astype(np.float64), axis=1) > 1.1 * R0
    assert floater.sum() > 0
    cx, _, cn, index = extract.clean_point_cloud(xyz, rgb, normals)
    idx = index.cpu().numpy()
    assert not floater[idx].any()
    # pass 1 against float64; pass 2 against float64 on the device's own survivors, which differ from float64's only
    # at flagged pass-1 decisions
    r1 = C.statistical64(x_np, 50)
    avg, keep, _ = device_stat(xyz, 50)
    C.check_statistical(avg, keep, r1, REPORT)
    moved1 = np.nonzero(keep != r1["keep"])[0]
    first = np.nonzero(keep)[0]
    r2 = C.normal64(x_np[first], n_np[first])
    mean, keep2 = device_angle(cu(x_np[first]), cu(n_np[first]), 20)
    C.check_normal(mean, keep2, r2, n_np[first], report=REPORT)
    assert np.array_equal(idx, first[keep2])  # the public function returns what the two checked passes decided
    # against float64's own two passes: any difference is a flagged element, or a point with a flipped pass-1 point
    # among its 20 nearest (its float64 neighbourhood is then another one)
    want = C.clean64(x_np, n_np)[0]
    flagged = set(moved1.tolist()) | set(first[C.flag_normal(r2) | r2["tie"] | r2["dup"]].tolist())
    unexplained = np.array([i for i in np.setxor1d(idx, want) if i not in flagged], np.int64)
    if len(unexplained) and len(moved1):
        _, nb = R.knn64(x_np, 21, queries=unexplained)
        unexplained = unexplained[~np.isin(nb, moved1).any(1)]
    assert len(unexplained) == 0, f"{len(unexplained)} kept / dropped points differ from float64 unflagged"
    print(f"end to end: {len(np.setxor1d(idx, want))} differences from float64, {len(moved1)} flipped pass-1 decisions")
    assert torch.isfinite(cn).all()
    v, f = extract.mesh_sap(cx, cn)
    dist = np.abs(np.linalg.norm(v.cpu().numpy().astype(np.float64), axis=1) - R0)
    print(f"{len(x_np)} fused, {int(floater.sum())} floaters, {len(idx)} kept, max |r - R| {dist.max():.4f}; {REPORT}")
    assert v.shape[0] > 0 and dist.max() < 0.02 * R0


def test_zz_report():
    print("clean report:", REPORT)
