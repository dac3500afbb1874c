"""-m gpu: Gaussian initialization on the device (gaustudio_b200.initializers, csrc/gsr_init.cu and MODE_DIST2 of
csrc/gsr_clean.cu) against the float64 restatements of tests/init_ref64.py: dist2 against cKDTree, the pcd
initializer against the reference's own torch code on the same device, the mesh initializer per row within bounds
derived per op, the occupied voxel set exactly, voxel colours against brute-force closest points; then a mesh2gs run
rendered, and a short fit started from the pcd initializer."""
import math

import numpy as np
import pytest
import torch

import init_ref64 as R
from gaustudio_b200 import initializers, io
from gaustudio_b200.synthetic import GaussianPointCloud

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
EPS = 2.0 ** -24


def cu(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dtype)


def uv_sphere(n_lat=24, n_lon=48, r=0.5, centre=(0.1, -0.2, 0.3), seed=0):
    """Closed UV sphere (poles shared) with smooth vertex colours -> (vertices float32, faces int64, colors)."""
    th = np.linspace(0, np.pi, n_lat + 1)[1:-1]
    ph = np.linspace(0, 2 * np.pi, n_lon, endpoint=False)
    T, P = np.meshgrid(th, ph, indexing="ij")
    v = np.stack([np.sin(T) * np.cos(P), np.sin(T) * np.sin(P), np.cos(T)], -1).reshape(-1, 3)
    v = np.concatenate([[[0, 0, 1]], v, [[0, 0, -1]]]) * r + np.asarray(centre)
    f = []
    idx = lambda i, j: 1 + i * n_lon + j % n_lon
    for j in range(n_lon):
        f.append([0, idx(0, j), idx(0, j + 1)])
        f.append([len(v) - 1, idx(n_lat - 2, j + 1), idx(n_lat - 2, j)])
    for i in range(n_lat - 2):
        for j in range(n_lon):
            f.append([idx(i, j), idx(i + 1, j), idx(i + 1, j + 1)])
            f.append([idx(i, j), idx(i + 1, j + 1), idx(i, j + 1)])
    col = 0.5 + 0.5 * np.stack([np.sin(3 * v[:, 0]), np.cos(2 * v[:, 1]), np.sin(v[:, 2] * 5)], 1)
    return v.astype(np.float32), np.array(f, np.int64), col.astype(np.float32)


def surface_cloud(n, seed, floaters=0.0):
    g = np.random.default_rng(seed)
    d = g.normal(size=(n, 3))
    x = 0.5 * d / np.linalg.norm(d, axis=1, keepdims=True)
    k = int(floaters * n)
    if k:
        x[:k] = g.uniform(-50, 50, (k, 3))
    return x.astype(np.float32)


# ---- dist2 ----
def check_dist2(x):
    got = initializers.dist2(cu(x)).cpu().numpy().astype(np.float64)
    ref = R.dist2_64(x)
    # the selection is float64's exactly; the mean is rounded once to float32 (plus two double roundings)
    fin = np.isfinite(ref)
    assert (np.isinf(got) == ~fin).all()
    assert (np.abs(got[fin] - ref[fin]) <= ref[fin] * (EPS + 1e-15)).all(), np.abs(got[fin] - ref[fin]).max()
    return got


@pytest.mark.parametrize("case", ["uniform", "surface", "duplicates", "floaters_1M"])
def test_dist2_against_ckdtree(case):
    g = np.random.default_rng(1)
    if case == "uniform":
        x = g.uniform(-1, 1, (50_000, 3)).astype(np.float32)
    elif case == "surface":
        x = surface_cloud(200_000, 2)
    elif case == "duplicates":
        x = g.uniform(-1, 1, (20_000, 3)).astype(np.float32)
        x[10_000:] = x[:10_000]
        x[:5] = x[5]
    else:
        x = surface_cloud(1_000_000, 3, floaters=0.01)
    got = check_dist2(x)
    if case == "duplicates":
        assert (got[:5] == 0).all()
    again = initializers.dist2(cu(x)).cpu().numpy().astype(np.float64)
    assert np.array_equal(got.view(np.int64), again.view(np.int64))


@pytest.mark.parametrize("n", [1, 2, 3, 4])
def test_dist2_tiny_clouds(n):
    x = np.arange(3 * n, dtype=np.float32).reshape(n, 3) ** 1.5
    got = check_dist2(x)
    assert np.isinf(got).all() == (n <= 3)


def test_dist2_refusals_and_drop_in():
    for bad in (np.nan, np.inf):
        x = np.zeros((10, 3), np.float32)
        x[3, 1] = bad
        with pytest.raises(ValueError):
            initializers.dist2(cu(x))
    assert initializers.dist2(torch.zeros(0, 3, device=DEV)).shape == (0,)
    from simple_knn._C import distCUDA2
    x = cu(surface_cloud(5000, 4))
    assert torch.equal(distCUDA2(x), initializers.dist2(x))


# ---- create_from_attribute / pcd ----
def reference_pcd(xyz, rgb, normals, sh_degree):
    """pcd.py:58-77 + vanilla_sg.py:69-97 as the reference computes them, on this device (its dist2 from cKDTree)."""
    x = torch.tensor(xyz, dtype=torch.float32).to(DEV)
    rgb = torch.ones_like(x) if rgb is None else torch.tensor(rgb, dtype=torch.float32).to(DEV)
    f_dc = ((rgb - 0.5) / R.SH_C0).unsqueeze(-1).transpose(1, 2)
    d2 = torch.tensor(R.dist2_64(x.cpu().numpy()), dtype=torch.float32, device=DEV)
    scale = torch.log(torch.sqrt(d2 + 1e-7))[..., None].repeat(1, 3)
    if normals is None:
        rot = torch.zeros(len(x), 4, device=DEV)
        rot[:, 0] = 1
    else:
        rot = R.normal2rotation_torch32(torch.tensor(normals).float().to(DEV))
    op = torch.tensor(np.log(0.1 * np.ones((len(x), 1)) / (1 - 0.1 * np.ones((len(x), 1)))), dtype=torch.float32)
    return dict(_xyz=x, _f_dc=f_dc, _scale=scale, _rot=rot, _opacity=op.to(DEV),
                _f_rest=torch.zeros(len(x), (sh_degree + 1) ** 2 - 1, 3, device=DEV))


@pytest.mark.parametrize("colors,normals", [(True, True), (False, False), (True, "zero"), (False, True)])
def test_pcd_initializer_against_reference(tmp_path, colors, normals):
    g = np.random.default_rng(5)
    n = 3000
    xyz = surface_cloud(n, 6).astype(np.float64)
    rgb = g.random((n, 3)) if colors else None
    nr = None
    if normals is True:
        nr = g.normal(size=(n, 3))
        nr[:40, 2] = 0
    elif normals == "zero":
        nr = np.zeros((n, 3))
    p = str(tmp_path / "points3D.ply")
    io.export_points_ply(p, xyz, rgb, nr)
    v = io.read_ply_vertices(p)
    rgb_read = None if rgb is None else np.stack([v[k] for k in ("red", "green", "blue")], 1) / 255.0
    model = initializers.make({"name": "pcd", "model_path": p})(GaussianPointCloud.empty(sh_degree=3))
    ref = reference_pcd(xyz, rgb_read, nr, 3)
    for k in ("_xyz", "_f_dc", "_f_rest", "_opacity"):
        assert torch.equal(getattr(model, k), ref[k]), k
    # the scale: float64's neighbour set, one float32 rounding of the mean, then float32 sqrt / log
    assert (model._scale - ref["_scale"]).abs().max() <= 4e-7 * (1 + ref["_scale"].abs().max())
    if nr is None:
        assert torch.equal(model._rot, ref["_rot"])
    else:
        q64, r, s, *_ = R.normal2rotation64(nr.astype(np.float32).astype(np.float64))
        err = np.abs(model._rot.cpu().numpy() - q64)
        assert (err <= R.quat_bound(q64, r, s)).all()
        if normals == "zero":
            assert torch.equal(model._rot, ref["_rot"])
            assert torch.allclose(torch.nn.functional.normalize(model._rot),
                                  torch.tensor([1.0, 0, 0, 0], device=DEV).expand(n, 4))
    out = str(tmp_path / "init.ply")
    io.export_ply(model, out)
    back = io.load_ply(out, sh_degree=3, device=DEV)
    assert torch.equal(back._xyz, model._xyz) and torch.equal(back._scale, model._scale)
    assert torch.equal(back._rot, model._rot) and torch.equal(back._opacity, model._opacity)
    assert torch.equal(back._f_dc.reshape(n, 3), model._f_dc.reshape(n, 3))


def test_create_from_attribute_empty():
    m = GaussianPointCloud.empty(sh_degree=1).create_from_attribute(np.zeros((0, 3)))
    assert m._xyz.shape == (0, 3) and m._scale.shape == (0, 3) and m._rot.shape == (0, 4) and m.num_points == 0


# ---- mesh ----
def test_vertex_normals_against_float64():
    v, f, _ = uv_sphere()
    got = initializers.vertex_normals(cu(v), cu(f, torch.int64)).cpu().numpy()
    ref = R.vertex_normals64(v, f)
    assert np.abs(got - ref).max() <= 4 * EPS


def mesh_rows(n, v, f, col):
    m = initializers.make({"name": "mesh", "n_gaussians_per_surface_triangle": n})
    return m(GaussianPointCloud.empty(sh_degree=1),
             (cu(v), cu(f, torch.int64), None if col is None else cu(col)))


@pytest.mark.parametrize("n", [1, 3, 4, 6])
def test_mesh_initializer_rows_against_float64(n):
    v, f, col = uv_sphere(16, 32)
    f = np.concatenate([f, [[0, 0, 5], [7, 7, 7]]])  # degenerate faces: a zero edge, then one point
    model = mesh_rows(n, v, f, col)
    vn = R.vertex_normals64(v, f).astype(np.float32)
    s = R.sugar64(v, f, vn, col, n)
    P = len(f) * n
    xyz = model._xyz.cpu().numpy()
    vmax = np.abs(v).max()
    assert np.abs(xyz - s["xyz"]).max() <= 3 * EPS * vmax * 2  # three products and two sums of float32 values
    rgb = model._f_dc.reshape(P, 3).cpu().numpy() * R.SH_C0 + 0.5
    assert np.abs(rgb - s["rgb"]).max() <= 1e-6
    sc = model._scale.cpu().numpy()
    ok = s["min_edge"] > 0
    # log(2 m r + 1e-7): the relative float32 error of m r (norm, product: ~4 eps) becomes an absolute one
    assert np.abs(sc[ok, 0] - s["scale_xy"][ok]).max() <= 8 * EPS + 1e-6
    assert np.array_equal(sc[:, 0], sc[:, 1])
    assert (sc[:, 2] == np.float32(np.log(np.float32(1e-7)))).all()
    assert (sc[~ok, 0] == sc[~ok, 2]).all()  # a zero edge: log(1e-7)
    assert torch.isinf(model._opacity).all() and (model._opacity > 0).all()
    q = model._rot.cpu().numpy()
    live = np.linalg.norm(s["normal"], axis=1) > 0.5
    q64, r, sn, R0, R1, nn = R.normal2rotation64(s["normal"])
    # flag rows whose sign decisions (R0_x, R1_y, n_z) lie within float32 rounding of 0
    near = (np.abs(R0[:, 0]) < 1e-5) | (np.abs(R1[:, 1]) < 1e-5) | (np.abs(nn[:, 2]) < 1e-5)
    bound = R.quat_bound(q64, r, sn) + 8 * EPS / (r[:, None] * np.minimum(sn, 1)[:, None])  # interpolated normal
    bad = (np.abs(q - q64) > bound).any(1) & live & ~near
    assert not bad.any(), (np.argwhere(bad)[:5], near.sum())
    again = mesh_rows(n, v, f, col)
    for k in ("_xyz", "_rot", "_f_dc", "_scale"):
        assert torch.equal(getattr(model, k), getattr(again, k))


def test_mesh_initializer_without_colours_is_white():
    v, f, _ = uv_sphere(8, 16)
    model = mesh_rows(3, v, f, None)
    # RGB2SH(1) as create_from_attribute computes it on the device, bit for bit
    assert torch.equal(model._f_dc, (torch.ones_like(model._f_dc) - 0.5) / R.SH_C0)


# ---- voxel ----
def voxel_case(name):
    if name == "sphere":
        v, f, c = uv_sphere(20, 40)
        return v, f, c
    if name == "cube":  # faces on cell faces after normalisation (extent 1, a multiple of 1/8)
        v = np.array([[x, y, z] for x in (0, 1) for y in (0, 1) for z in (0, 1)], np.float32)
        f = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6],
                      [0, 2, 6], [0, 6, 4], [1, 5, 7], [1, 7, 3]], np.int64)
        return v, f, np.random.default_rng(0).random((8, 3)).astype(np.float32)
    if name == "slivers":
        g = np.random.default_rng(7)
        a = g.uniform(-1, 1, (60, 3))
        b = a + g.normal(size=(60, 3)) * 0.5
        c = a + (b - a) * g.random((60, 1)) + g.normal(size=(60, 3)) * 1e-4
        v = np.stack([a, b, c], 1).reshape(-1, 3).astype(np.float32)
        return v, np.arange(len(v)).reshape(-1, 3), g.random((len(v), 3)).astype(np.float32)
    if name == "zero_edge":  # one face with two coincident vertices, alone in the grid
        v = np.array([[-0.3, -0.2, 0.1], [-0.3, -0.2, 0.1], [0.4, 0.3, -0.2]], np.float32)
        return v, np.array([[0, 1, 2]]), np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    if name == "collinear":  # exactly collinear float32 faces; the box is not dyadic, so normalising breaks that
        g = np.random.default_rng(8)
        a = g.integers(-40, 40, (30, 3)) / 64.0
        d = g.integers(-20, 21, (30, 3)) / 128.0
        v = np.stack([a, a + d, a + g.integers(1, 4, (30, 1)) * d], 1).reshape(-1, 3)
        v = np.concatenate([v, [[0.31, -0.27, 1.113], [0.32, -0.27, 1.113], [0.31, -0.26, 1.113]]]).astype(np.float32)
        return v, np.arange(len(v)).reshape(-1, 3), g.random((len(v), 3)).astype(np.float32)
    if name == "spanning":
        v = np.array([[-1, -1, -1], [1, 1, -0.2], [-0.3, 1, 1]], np.float32)
        return v, np.array([[0, 1, 2]]), np.eye(3, dtype=np.float32)
    raise KeyError(name)


@pytest.mark.parametrize("name", ["sphere", "cube", "slivers", "zero_edge", "collinear", "spanning"])
@pytest.mark.parametrize("vs", [1 / 256, 0.01])
def test_voxel_occupied_set_and_colours(name, vs):
    v, f, col = voxel_case(name)
    init = initializers.make({"name": "voxel", "voxel_size": vs})
    vn, centre, scale = initializers.normalize_mesh(cu(v))
    cells, off, tris = initializers.voxelize(vn, cu(f, torch.int64), init.res, vs)
    vn64 = vn.cpu().numpy()
    ref = R.occupied64(vn64, f, init.res, vs)
    assert np.array_equal(cells.cpu().numpy().astype(np.int64), ref)
    model = init(GaussianPointCloud.empty(sh_degree=0), (cu(v), cu(f, torch.int64), cu(col)),
                 generator=torch.Generator().manual_seed(3))
    U = len(ref)
    assert model._xyz.shape == (U, 3)
    ijk = np.stack([ref // init.res ** 2, ref // init.res % init.res, ref % init.res], 1)
    ctr = R.voxel_centres(ijk, vs)
    np.testing.assert_array_equal(model._xyz.cpu().numpy(),
                                  (ctr * float(scale) + centre.cpu().numpy()).astype(np.float32))
    # colours against brute force over every triangle, for a sample of voxels; near-ties flagged
    g = np.random.default_rng(0)
    rgb = model._f_dc.reshape(U, 3).cpu().numpy() * R.SH_C0 + 0.5
    flagged = 0
    for i in g.choice(U, min(U, 300), replace=False):
        d = np.array([R.closest_bary64(ctr[i], *vn64[t])[0] for t in f])
        order = np.argsort(d, kind="stable")
        t = order[0]
        if len(d) > 1 and d[order[1]] - d[t] <= 1e-12 * (1 + d[t]):  # a gap within double rounding: either may win
            flagged += 1
            continue
        bc = R.closest_bary64(ctr[i], *vn64[f[t]])[1]
        want = bc @ col[f[t]].astype(np.float64)
        assert np.abs(rgb[i] - want).max() <= 1e-6, (i, rgb[i], want)
    sc = model._scale.cpu().numpy()
    assert (sc == np.float32(np.log(np.float32(vs * float(scale) * 0.8) + np.float32(1e-7)))).all()
    assert torch.isinf(model._opacity).all()
    again = init(GaussianPointCloud.empty(sh_degree=0), (cu(v), cu(f, torch.int64), cu(col)),
                 generator=torch.Generator().manual_seed(3))
    assert torch.equal(again._rot, model._rot) and torch.equal(again._f_dc, model._f_dc)
    assert torch.allclose(model._rot.norm(dim=1), torch.ones(U, device=DEV))


def test_voxelize_double_rounded_collinear_faces():
    """Faces collinear up to the rounding of t0 + s e in double, whose computed normals are rounding noise: the
    occupied set is still tribox3's."""
    g = np.random.default_rng(9)
    t0, e = g.uniform(-0.4, 0.4, (200, 3)), g.uniform(-1, 1, (200, 3)) * 0.1
    v = np.stack([t0, t0 + e, t0 + 0.37 * e], 1).reshape(-1, 3)
    f = np.arange(len(v)).reshape(-1, 3)
    cells, _, _ = initializers.voxelize(cu(v, torch.float64), cu(f, torch.int64), 256, 1 / 256)
    assert np.array_equal(cells.cpu().numpy().astype(np.int64), R.occupied64(v, f, 256, 1 / 256))


def test_voxel_without_colours_is_white():
    v, f, _ = voxel_case("cube")
    model = initializers.make({"name": "voxel", "voxel_size": 1 / 16})(GaussianPointCloud.empty(),
                                                                        (cu(v), cu(f, torch.int64), None))
    assert torch.equal(model._f_dc, (torch.ones_like(model._f_dc) - 0.5) / R.SH_C0)


# ---- end to end ----
def test_mesh2gs_flow_renders_opaque(tmp_path):
    from gaustudio_b200 import mesh as M, renderers
    from gaustudio_b200.camera import orbit_cameras
    v, f, col = uv_sphere(48, 96, centre=(0, 0, 0))
    p = str(tmp_path / "sphere.ply")
    io.export_mesh_ply(p, v, f, col)
    model = initializers.make({"name": "mesh", "n_gaussians_per_surface_triangle": 3})(
        GaussianPointCloud.empty(sh_degree=1), p)
    out = str(tmp_path / "gs.ply")
    io.export_ply(model, out)
    back = io.load_ply(out, sh_degree=1, device=DEV)
    assert torch.equal(back._xyz, model._xyz) and torch.isinf(back._opacity).all()
    vv, ff, _ = io.load_mesh_ply(p, device=DEV)
    for name in ("vanilla_renderer",):
        for fused in (False, True):
            r = renderers.make({"name": name, "fused_activations": fused})
            for cam in orbit_cameras(3, 2.0, 20.0, 96, 96, 0.8, 0.8):
                cam = cam.to(DEV)
                with torch.no_grad():
                    o = r.render(cam, back)
                img, op = o["render"], o["rendered_final_opacity"][0]
                assert torch.isfinite(img).all() and torch.isfinite(op).all()
                face, _ = M.rasterize(vv, ff, cam)
                cov = face >= 0
                assert cov.sum() > 500
                assert float((op[cov] > 0.5).float().mean()) >= 0.99


def test_fit_from_pcd_initializer(tmp_path):
    from gaustudio_b200 import densify, extract, optimizers, renderers
    from gaustudio_b200.camera import orbit_cameras
    v, f, col = uv_sphere(48, 96, centre=(0, 0, 0))
    gt = initializers.make({"name": "mesh", "n_gaussians_per_surface_triangle": 3})(
        GaussianPointCloud.empty(sh_degree=0), (cu(v), cu(f, torch.int64), cu(col)))
    cams = [c.to(DEV) for c in orbit_cameras(8, 2.0, 20.0, 80, 80, 0.8, 0.8)]
    r = renderers.make({"name": "vanilla_renderer"})
    with torch.no_grad():
        targets = [r.render(c, gt)["render"].clone() for c in cams]
    g = np.random.default_rng(9)
    d = g.normal(size=(2000, 3))
    pts = 0.5 * d / np.linalg.norm(d, axis=1, keepdims=True)
    p = str(tmp_path / "points3D.ply")
    io.export_points_ply(p, pts, 0.5 + 0 * pts, pts)
    model = initializers.make({"name": "pcd", "model_path": p})(GaussianPointCloud.empty(sh_degree=0))
    for k in model._ATTRS:
        setattr(model, k, torch.nn.Parameter(getattr(model, k).contiguous()))
    lrs = (1.6e-4, 5e-3, 1e-3, 5e-2, 2.5e-3, 1.25e-4)
    opt = optimizers.FusedAdam([{"params": [p], "lr": lr} for p, lr in zip(model.parameters_list(), lrs)],
                               eps=1e-15, weight_decay=0.0)
    extent = extract.getNerfppNorm(cams)["radius"]
    losses = []
    for it in range(200):
        k = it % len(cams)
        o = r.render(cams[k], model)
        loss = (o["render"] - targets[k]).abs().mean()
        loss.backward()
        densify.add_densification_stats(model, o)
        opt.step(zero_grad=True)
        losses.append(float(loss))
        if (it + 1) % 50 == 0 and it + 1 < 200:
            grad = (model.xyz_gradient_accum / model.denom).nan_to_num(0.0)
            densify.densify_and_prune(model, opt, float(torch.quantile(grad[grad > 0], 0.8)), 0.005, extent, None)
    assert all(bool(torch.isfinite(p).all()) for p in model.parameters_list())
    first, last = np.mean(losses[:8]), np.mean(losses[-8:])
    assert last < 0.8 * first, (first, last)
