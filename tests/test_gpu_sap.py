"""-m gpu: Shape-as-Points meshing on the device (extract.dpsr / extract.mesh_sap, csrc/gsr_sap.cu) against the float64
restatement of tests/sap_ref64.py, with no outlier budget: the splat per node, psi at res 32 / 128 / 256, bitwise
repeatability, independence from what the allocator's blocks held, the meshes of the golden shapes, degenerate point
sets, and the whole extract_pcd -> mesh_sap flow on a rendered sphere."""
import math
import os

import numpy as np
import pytest
import torch

import sap_ref64 as S
from gaustudio_b200 import _lib, extract

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
U = S.U32
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sap_golden.npz")


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(DEV)


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


def splat_bound(p, n, res):
    """Each term w_x w_y w_z n is a float32 product of float32 weights (one division, one subtraction and one
    division per axis): <= 12 u |term|; the node sums those terms in double and rounds once (u |sum|)."""
    g, mag = S.splat64(p, n, res)
    return g, 12.0 * U * mag[None] + U * np.abs(g) + 1e-38


def normalize_on_device(xyz):
    """gsr_sap_normalize as mesh_sap calls it -> (points01, transform (c, s))."""
    p = torch.empty_like(xyz)
    t = torch.empty(4, dtype=torch.float32, device=DEV)
    with _lib.scratch(DEV):
        _lib.call("gsr_sap_normalize", DEV, xyz.shape[0], _lib.ptr(xyz), _lib.ALLOC, 1, _lib.ptr(p), _lib.ptr(t))
    return p, t


@pytest.mark.parametrize("shape", list(S.SHAPES))
@pytest.mark.parametrize("res", [32, 64, 128])
def test_splat_per_node_against_float64(gold, shape, res):
    p, n = gold[f"{shape}_p"], gold[f"{shape}_normals"]
    g = extract._sap_splat(cu(p), cu(n), res).cpu().numpy()
    want, bound = splat_bound(p.astype(np.float64), n, res)
    assert (np.abs(g - want) <= bound).all(), (np.abs(g - want) / bound).max()
    np.testing.assert_allclose(g.reshape(3, -1).astype(np.float64).sum(1), n.astype(np.float64).sum(0),
                               rtol=0, atol=1e-5 * np.abs(n).sum())


def test_splat_wrap_and_on_node_points():
    res = 16
    p = np.array([[15.25, 3.0, 7.5], [0.0, 15.0, 15.5], [4.0, 4.0, 4.0], [15.75, 15.75, 15.75]]) / res
    n = np.array([[1.0, -2.0, 0.5], [0.3, 0.4, -1.0], [2.0, 1.0, 1.0], [-1.0, 1.0, 3.0]])
    g = extract._sap_splat(cu(p), cu(n), res).cpu().numpy()
    want, bound = splat_bound(p, n, res)
    assert (np.abs(g - want) <= bound).all()
    assert g[0, 0, 3, 7] == np.float32(0.25 * 0.5 * 1.0) and g[:, 4, 4, 4].tolist() == [2.0, 1.0, 1.0]


def _psi_case(gold, shape, res):
    xyz, n = gold[f"{shape}_p"], gold[f"{shape}_normals"]  # the golden points, taken as world coordinates
    p, _, _ = S.normalize64(xyz)
    p = p.astype(np.float32)
    return p, n, S.dpsr64(p.astype(np.float64), n, res)


@pytest.mark.parametrize("res", [32, 128, 256])
@pytest.mark.parametrize("shape", ["sphere", "torus"])
def test_psi_against_float64(gold, shape, res):
    """Bound: sap_ref64.psi_bound (float32 splat and FFTs, carried through the shift, the scale and the tanh)."""
    p, n, ref = _psi_case(gold, shape, res)
    psi = extract.dpsr(cu(p), cu(n), res=res).cpu().numpy()
    err, tol = np.abs(psi - ref["psi"]).max(), S.psi_bound(ref, res)
    print(f"{shape} res {res}: max|psi - psi64| = {err:.3e}, bound {tol:.3e} ({err / tol:.3f} of it), "
          f"max|psi| {np.abs(ref['psi']).max():.3f}")
    assert err <= tol


def test_same_bits_on_two_runs(gold):
    xyz, n = cu(gold["torus_p"]), cu(gold["torus_normals"])
    a, b = extract.mesh_sap(xyz, n, res=128), extract.mesh_sap(xyz, n, res=128)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    p, _ = normalize_on_device(xyz)
    assert torch.equal(extract.dpsr(p, n, res=96), extract.dpsr(p, n, res=96))
    assert torch.equal(extract._sap_splat(p, n, 200), extract._sap_splat(p, n, 200))


def test_results_do_not_depend_on_what_the_allocator_held(gold):
    xyz, n = cu(gold["sphere_p"]), cu(gold["sphere_normals"])
    torch.cuda.empty_cache()
    clean = extract.mesh_sap(xyz, n, res=128)
    junk = [torch.full((k,), float("nan"), device=DEV) for k in (1 << 10, 1 << 16, 1 << 20, 1 << 22, 1 << 24, 1 << 25)]
    junk += [torch.full((1 << 22,), -7, dtype=torch.int32, device=DEV) for _ in range(4)]
    del junk  # the caching allocator keeps these blocks and hands them out again
    again = extract.mesh_sap(xyz, n, res=128)
    assert torch.equal(clean[0], again[0]) and torch.equal(clean[1], again[1])


@pytest.mark.parametrize("shape", list(S.SHAPES))
def test_mesh_of_golden_shapes(gold, shape):
    res = 64
    xyz_np, n_np = gold[f"{shape}_p"], gold[f"{shape}_normals"]  # the golden points, taken as world coordinates
    xyz, n = cu(xyz_np), cu(n_np)
    v, f = extract.mesh_sap(xyz, n, res=res)
    v, f = v.cpu().numpy().astype(np.float64), f.cpu().numpy()
    assert len(f) > 0 and f.min() >= 0 and f.max() < len(v) and len(np.unique(f)) == len(v)
    # every vertex on the zero level of the device's own trilinear psi: a vertex is the linear zero crossing of an
    # edge, where trilinear interpolation is linear; its float32 world coordinates, mapped back, move it by <= 16 u res
    # index units, and psi changes by at most L per unit there (L: largest difference of neighbouring nodes)
    p, t = normalize_on_device(xyz)
    psi = extract.dpsr(p, n, res=res).cpu().numpy().astype(np.float64)
    c, s = t[:3].cpu().numpy().astype(np.float64), float(t[3])
    q = ((v - c) / s + 1.0) / 2.0 * res
    L = max(np.abs(np.diff(psi, axis=a)).max() for a in range(3))
    lvl = np.abs(S.trilinear(psi, q)).max()
    assert lvl <= 16 * U * res * L * math.sqrt(3) + 1e-7, (lvl, L)
    # against the float64 restatement's mesh
    v64, f64, ref, _, s64 = S.mesh64(xyz_np, n_np, res)
    voxel = 2.0 * s64 / res
    ch = S.chamfer(v, v64)
    print(f"{shape}: V {len(v)} / {len(v64)}, F {len(f)} / {len(f64)}, chamfer {ch / voxel:.2e} voxel, level {lvl:.1e}")
    assert ch < 0.5 * voxel
    if shape == "sphere":
        closed, euler = S.edge_manifold(f)
        assert closed and euler == 2
        centre = xyz_np.astype(np.float64).mean(0)
        nrm = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
        assert (np.einsum("ij,ij->i", nrm, v[f].mean(1) - centre) > 0).all()


def test_sphere_at_res_256_is_closed_outward_and_at_its_radius():
    centre, r = np.array([0.1, -0.2, 0.3]), 0.5
    xyz, n = S.sphere(200_000, r=r, centre=centre, seed=5)
    v, f = extract.mesh_sap(cu(xyz), cu(n))
    v, f = v.cpu().numpy().astype(np.float64), f.cpu().numpy()
    s = 1.2 * np.abs(xyz.astype(np.float64) - xyz.mean(0)).max()
    assert np.abs(np.linalg.norm(v - centre, axis=1) - r).max() < 2.0 * s / 256
    closed, euler = S.edge_manifold(f)
    assert closed and euler == 2
    nrm = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    assert (np.einsum("ij,ij->i", nrm, v[f].mean(1) - centre) > 0).all()


@pytest.mark.parametrize("case", ["one_point", "one_cell"])
def test_degenerate_point_sets(case):
    res = 32
    g = np.random.default_rng(3)
    if case == "one_point":
        p, n = np.array([[0.4, 0.55, 0.61]]), np.array([[0.0, 0.6, 0.8]])
    else:  # 1000 points inside cell (12, 20, 7)
        p = (np.array([12, 20, 7]) + g.uniform(0.01, 0.99, (1000, 3))) / res
        n = g.normal(size=(1000, 3))
    p, n = p.astype(np.float32), n.astype(np.float32)
    ref = S.dpsr64(p.astype(np.float64), n, res)
    psi = extract.dpsr(cu(p), cu(n), res=res).cpu().numpy()
    assert np.abs(psi - ref["psi"]).max() <= S.psi_bound(ref, res)
    grid = extract._sap_splat(cu(p), cu(n), res).cpu().numpy()
    want, bound = splat_bound(p.astype(np.float64), n, res)
    assert (np.abs(grid - want) <= bound).all() and np.count_nonzero(grid[0]) <= 8


def test_device_refusals():
    ok = torch.rand(10, 3, device=DEV)
    with pytest.raises(ValueError, match="finite"):
        extract.dpsr(torch.full((10, 3), float("nan"), device=DEV), ok)
    with pytest.raises(ValueError, match="finite"):
        extract.mesh_sap(ok, torch.full((10, 3), float("inf"), device=DEV))
    with pytest.raises(ValueError, match=r"\[0, 1\)"):
        extract.dpsr(ok + 1.0, ok)
    with pytest.raises(ValueError, match=r"\[0, 1\)"):
        extract.dpsr(ok - 1.0, ok)
    with pytest.raises(ValueError, match="distinct"):
        extract.mesh_sap(torch.ones(5, 3, device=DEV), torch.rand(5, 3, device=DEV))


def test_extract_pcd_then_mesh_sap_lies_on_the_rendered_sphere():
    """A sphere of radius R covered by small opaque Gaussians, seen from two orbits: the fused points are Gaussian
    centres on the sphere, so the mesh must lie within 2 % of R of it (about 2.3 voxels at res 256)."""
    from gaustudio_b200 import renderers
    from gaustudio_b200.camera import orbit_cameras
    from gaustudio_b200.synthetic import GaussianPointCloud
    R, P = 0.6, 60_000
    g = torch.Generator().manual_seed(7)
    d = torch.randn(P, 3, generator=g)
    d = d / d.norm(dim=1, keepdim=True)
    pcd = GaussianPointCloud(R * d, torch.full((P, 3), math.log(0.012)), torch.randn(P, 4, generator=g),
                             torch.full((P, 1), 4.0), torch.randn(P, 1, 3, generator=g), torch.zeros(P, 15, 3), 3, 0)
    pcd.to(DEV)
    fov = math.radians(40.0)
    cams = orbit_cameras(16, 2.5, 35.0, 160, 160, fov, fov) + orbit_cameras(16, 2.5, -35.0, 160, 160, fov, fov)
    cams = [c.to(DEV) for c in cams]
    xyz, _, normals, _ = extract.extract_pcd(renderers.make({"name": "vanilla_renderer"}), pcd, cams)
    keep = ~torch.isnan(normals).any(1)
    xyz, normals = xyz[keep].detach().float().contiguous(), normals[keep].float().contiguous()
    assert xyz.shape[0] > 1000
    v, f = extract.mesh_sap(xyz, normals)
    dist = np.abs(np.linalg.norm(v.cpu().numpy().astype(np.float64), axis=1) - R)
    print(f"{xyz.shape[0]} points, V {v.shape[0]}, F {f.shape[0]}, max |r - R| {dist.max():.4f}, "
          f"median {np.median(dist):.5f}")
    assert v.shape[0] > 0 and dist.max() < 0.02 * R
