"""CPU checks of the Gaussian initializers: the float64 restatements of tests/init_ref64.py against independent
brute-force or exact versions, and every refusal of the Python surface before any device work."""
import math

import numpy as np
import pytest
import torch

import init_ref64 as R
from gaustudio_b200 import _lib, initializers
from gaustudio_b200.synthetic import GaussianPointCloud


def test_tribox_matches_exact_test_on_random_triangles():
    g = np.random.default_rng(0)
    for _ in range(4000):
        t = g.uniform(-1.5, 1.5, (3, 3)) * g.choice([0.05, 0.5, 2.0])
        c = g.uniform(-1, 1, 3) * 0.5
        h = float(g.choice([0.125, 0.25, 0.5]))
        assert R.tribox64(c[None], h, t[None])[0] == R.tribox_exact(c, h, t)


def test_tribox_touching_dyadic_cases_agree_exactly():
    """Triangles on grid planes and through box edges and corners, with dyadic coordinates: float64 is exact there,
    so the restatement must give exactly the exact test's answer, touches counting as overlap."""
    g = np.random.default_rng(1)
    h = 0.125
    n_touch = 0
    for _ in range(3000):
        c = g.integers(-4, 5, 3) * 0.25
        t = g.integers(-12, 13, (3, 3)) * 0.0625 + c
        # push one coordinate of every vertex onto a face plane of the box, or a vertex onto a corner
        kind = g.integers(0, 3)
        if kind == 0:
            d = g.integers(0, 3)
            t[:, d] = c[d] + h * g.choice([-1, 1])
        elif kind == 1:
            t[0] = c + h * g.choice([-1, 1], 3)
        exact = R.tribox_exact(c, h, t)
        assert R.tribox64(c[None], h, t[None])[0] == exact
        n_touch += exact
    assert n_touch > 100


def test_cube_on_cell_faces_occupies_both_sides():
    """A face lying on a cell face touches the cells on both sides (tribox3 counts a touch)."""
    res, vs = 8, 1 / 8
    t = np.array([[[0.0, -0.25, -0.25], [0.0, 0.25, -0.25], [0.0, 0.25, 0.25]]])
    occ = R.occupied64(t[0], np.array([[0, 1, 2]]), res, vs)
    i = occ // (res * res)
    assert set(i.tolist()) == {3, 4}


def test_closest_point_against_brute_force():
    g = np.random.default_rng(2)
    for _ in range(3000):
        a, b, c = g.normal(size=(3, 3))
        if g.random() < 0.1:
            c = a + g.random() * (b - a)  # collinear
        p = g.normal(size=3) * 1.5
        d2, bc = R.closest_bary64(p, a, b, c)
        ref = R.closest_brute(p, a, b, c)
        assert abs(d2 - ref) <= 1e-9 * (1 + ref), (d2, ref)
        assert abs(bc.sum() - 1) < 1e-12 and (bc >= -1e-12).all()


def test_closest_point_of_zero_edge_faces_is_finite_and_exact():
    """a == b (a zero edge) and all three vertices equal: the distance is finite and equals brute force."""
    g = np.random.default_rng(6)
    a = np.array([-0.3, -0.2, 0.1]); c = np.array([0.4, 0.3, -0.2])
    for _ in range(2000):
        p = g.uniform(-0.6, 0.6, 3)
        for tri in ((a, a, c), (a, c, c), (c, a, a), (a, a, a)):
            d2, bc = R.closest_bary64(p, *tri)
            assert np.isfinite(d2) and np.isfinite(bc).all()
            assert abs(d2 - R.closest_brute(p, *tri)) <= 1e-12 * (1 + d2)


def _normalised(v):
    """normalize_mesh's double ops on float32 vertices."""
    v = np.asarray(v, np.float32).astype(np.float64)
    lo, hi = v.min(0), v.max(0)
    centre, scale = (lo + hi) / 2, (hi - lo).max()
    return np.clip((v - centre) / scale, -0.5 + 1e-6, 0.5 - 1e-6)


def _covers(t, res, vs):
    occ = R.occupied64(t, np.array([[0, 1, 2]]), res, vs)
    cand = R.candidates64(t, res, vs)
    ijk = {(int(x // (res * res)), int(x // res % res), int(x % res)) for x in occ}
    return ijk <= cand, len(ijk)


@pytest.mark.parametrize("vs", [1 / 256, 1 / 64])
def test_candidates_cover_every_occupied_cell_of_degenerate_faces(vs):
    """The kernel's candidate cells hold every cell tribox3 accepts, also for faces whose computed normal is rounding
    noise: exactly collinear float32 faces normalised with a non-dyadic bounding box, and collinear faces perturbed
    by 1e-15."""
    res = int(round(1 / vs))
    g = np.random.default_rng(7)
    n_occ = 0
    for it in range(90):
        if it % 3 == 0:  # exactly collinear in float32, normalised in double with a non-dyadic box
            a = g.integers(-40, 40, 3) / 64.0
            d = g.integers(-6, 7, 3) / 128.0
            v = np.stack([a, a + d, a + g.integers(1, 4) * d, g.uniform(-1, 1, 3) * 0.37 + 0.013])
            t = _normalised(v)[:3]
        elif it % 3 == 1:  # collinear up to the rounding of t0 + s e in double
            t0, e = g.uniform(-0.4, 0.4, 3), g.uniform(-1, 1, 3) * 0.1
            t = np.stack([t0, t0 + e, t0 + 0.37 * e])
        else:  # collinear faces perturbed by 1e-15
            t0, e = g.uniform(-0.4, 0.4, 3), g.uniform(-1, 1, 3) * 0.1
            t = np.stack([t0, t0 + e, t0 + 0.61 * e]) + g.normal(size=(3, 3)) * 1e-15
        ok, n = _covers(t, res, vs)
        assert ok, (it, t)
        n_occ += n
    assert n_occ > 500
    for _ in range(40):  # ordinary triangles
        t = g.uniform(-0.45, 0.45, (3, 3)) * g.choice([0.02, 0.2, 1.0])
        assert _covers(t, res, vs)[0]


def test_vertex_normals_and_sugar_restatements_against_per_face_loops():
    g = np.random.default_rng(3)
    v = g.normal(size=(30, 3))
    f = g.integers(0, 30, (60, 3))
    vn = R.vertex_normals64(v, f)
    acc = np.zeros_like(v)
    for i in range(len(f)):
        n = np.cross(v[f[i, 1]] - v[f[i, 0]], v[f[i, 2]] - v[f[i, 0]])
        for c in range(3):
            acc[f[i, c]] = acc[f[i, c]] + n
    for k in range(len(v)):
        l = np.linalg.norm(acc[k])
        np.testing.assert_allclose(vn[k], acc[k] / l if l > 0 else 0 * acc[k], rtol=0, atol=1e-12)
    col = g.random((30, 3))
    for n in (1, 3, 4, 6):
        s = R.sugar64(v, f, vn, col, n)
        assert s["xyz"].shape == (60 * n, 3)
        for i in (0, 17, 59):
            for j in range(n):
                b = np.float32(R.BARY[n][j]).astype(np.float64)
                np.testing.assert_allclose(s["xyz"][i * n + j], sum(b[c] * v[f[i, c]] for c in range(3)), atol=1e-12)
                e = min(np.linalg.norm(v[f[i, c]] - v[f[i, (c + 1) % 3]]) for c in range(3))
                assert s["scale_xy"][i * n + j] == pytest.approx(math.log(2 * e * R.RADIUS[n] + 1e-7), abs=1e-12)


def test_normal2rotation_float64_against_float32_torch():
    g = np.random.default_rng(4)
    n = g.normal(size=(5000, 3))
    n[:50, 2] = 0  # n_z = 0: R1 zeroed
    n[50:60] = 0   # all-zero (COLMAP-style) normals
    q64, r, s, *_ = R.normal2rotation64(n)
    q32 = R.normal2rotation_torch32(torch.from_numpy(n).float()).double().numpy()
    bad = np.abs(q32 - q64) > R.quat_bound(q64, r, s)
    # no sign decision of these normals lies within rounding of 0, so no row is exempt
    assert not bad.any(), np.argwhere(bad)[:5]
    np.testing.assert_allclose(q64[50:60], [[math.sqrt(2 + 1e-6) / 2, 0, 0, 0]] * 10, atol=0)
    nn = n[:50] / np.linalg.norm(n[:50], axis=1, keepdims=True)
    np.testing.assert_allclose(q64[:50, 1], -nn[:, 1] / (4 * r[:50]), rtol=1e-12)  # R1 = 0: x = (0 - n_y) / 4r


def test_registry_surface():
    assert {"pcd", "mesh", "voxel"} <= set(initializers.initializers)
    with pytest.raises(ValueError):
        initializers.make({})
    with pytest.raises(ValueError):
        initializers.make("no_such")
    assert initializers.make({"name": "mesh"}).n_gaussians_per_surface_triangle == 1
    assert initializers.make({"name": "mesh", "n_gaussians_per_surface_triangle": 3}).n_gaussians_per_surface_triangle == 3
    assert initializers.make({"name": "voxel", "voxel_size": 0.01}).res == 100


@pytest.mark.parametrize("n", [0, 2, 5, 7, 3.0, True, "3", None])
def test_bad_n_refused(n):
    with pytest.raises(ValueError):
        initializers.make({"name": "mesh", "n_gaussians_per_surface_triangle": n})


@pytest.mark.parametrize("vs", [0, -0.01, math.inf, math.nan, 1 / 2000, 3.0, True, "0.01"])
def test_bad_voxel_size_refused(vs):
    with pytest.raises(ValueError):
        initializers.make({"name": "voxel", "voxel_size": vs})


def _cpu_model():
    return GaussianPointCloud.empty(sh_degree=1, device="cpu")


def test_empty_model():
    m = GaussianPointCloud.empty(sh_degree=2, device="cpu")
    assert m.active_sh_degree == 0 and m.max_sh_degree == 2 and m.num_points == 0
    assert m._f_rest.shape == (0, 8, 3) and m.get_features.shape == (0, 9, 3)


def test_create_from_attribute_on_cpu_with_every_attribute():
    g = np.random.default_rng(5)
    P = 7
    xyz, rgb = g.normal(size=(P, 3)), g.random((P, 3))
    m = _cpu_model().create_from_attribute(xyz, rgb=rgb, scale=np.zeros((P, 3)), rot=torch.ones(P, 4),
                                           opacity=np.ones((P, 1)))
    assert m._xyz.dtype == torch.float32 and m._f_dc.shape == (P, 1, 3) and m._f_rest.shape == (P, 3, 3)
    np.testing.assert_array_equal(m._xyz.numpy(), xyz.astype(np.float32))
    ref = (torch.tensor(rgb, dtype=torch.float32) - 0.5) / R.SH_C0
    np.testing.assert_array_equal(m._f_dc[:, 0].numpy(), ref.numpy())
    assert m.num_points == P


def test_create_from_attribute_replaces_parameters():
    """A model set up for training (nn.Parameter attributes) can be initialised again: each attribute becomes a new
    Parameter holding the new values, with the same requires_grad."""
    m = _cpu_model().create_from_attribute(np.zeros((3, 3)), scale=np.zeros((3, 3)))
    for k in m._ATTRS:
        setattr(m, k, torch.nn.Parameter(getattr(m, k)))
    m._rot.requires_grad_(False)
    xyz = np.arange(15.0).reshape(5, 3)
    m.create_from_attribute(xyz, scale=np.ones((5, 3)))
    for k in m._ATTRS:
        assert isinstance(getattr(m, k), torch.nn.Parameter) and getattr(m, k).shape[0] == 5, k
    assert not m._rot.requires_grad and m._xyz.requires_grad
    np.testing.assert_array_equal(m._xyz.detach().numpy(), xyz.astype(np.float32))
    assert {n for n, _ in m.named_parameters()} == set(m._ATTRS)


def test_create_from_attribute_refusals_before_device_work():
    m = _cpu_model()
    P = 4
    with pytest.raises(ValueError, match="CPU path"):
        m.create_from_attribute(np.zeros((P, 3)))  # scale=None needs dist2
    ok = dict(scale=np.zeros((P, 3)))
    for bad in (dict(xyz=np.zeros((P, 2))), dict(xyz=np.zeros(P)), dict(xyz="abc"),
                dict(xyz=np.zeros((P, 3), complex)), dict(xyz=np.zeros((P, 3), bool))):
        with pytest.raises(ValueError):
            m.create_from_attribute(**{**ok, **bad})
    for bad in (dict(rgb=np.zeros((P, 4))), dict(rot=np.zeros((P, 3))), dict(opacity=np.zeros((P, 2))),
                dict(scale=np.zeros((P + 1, 3)))):
        with pytest.raises(ValueError):
            m.create_from_attribute(np.zeros((P, 3)), **{**ok, **bad})


def test_initializer_refusals_before_device_work(tmp_path):
    from gaustudio_b200 import io
    v = torch.tensor([[0.0, 0, 0], [1, 0, 0], [0, 1, 0]])
    f = torch.tensor([[0, 1, 2]])
    mesh = initializers.make({"name": "mesh"})
    cpu = _cpu_model()
    with pytest.raises(ValueError, match="CPU path"):
        mesh(cpu, (v, f, None))
    with pytest.raises(ValueError):
        mesh(cpu, (v.double(), f, None))
    with pytest.raises(ValueError):
        mesh(cpu, (v, f.int(), None))
    with pytest.raises(ValueError):
        mesh(cpu, (v, f, torch.ones(2, 3)))
    with pytest.raises(ValueError):
        mesh(cpu, (v, f[:0], None))
    with pytest.raises(ValueError):
        mesh(cpu, "not a mesh tuple".split())
    with pytest.raises(ValueError, match="CPU path"):
        initializers.make({"name": "voxel"})(cpu, (v, f, None))
    p = str(tmp_path / "p.ply")
    io.export_points_ply(p, np.zeros((4, 3)))
    with pytest.raises(ValueError, match="CPU path"):
        initializers.make({"name": "pcd", "model_path": p})(cpu)
    with pytest.raises(ValueError):
        initializers.dist2(torch.zeros(4, 3))
    with pytest.raises(ValueError):
        initializers.dist2(torch.zeros(4, 3, dtype=torch.float64))
    with pytest.raises(ValueError):
        initializers.normal2rotation(torch.zeros(4, 2))


# ---- refusals of the C entries: each check returns -1 with its text, before any device work ----
_NULL_FN = _lib.ALLOC_FN()
_FN = _lib.ALLOC_FN(lambda u, n: 0)
_P = 1 << 20  # fake device address, never dereferenced: every call below is refused before any work


def _range(what):
    return f"{what} must be in 1..2^31-1"


def _counts(*names):
    return [dict({k: 0 for k in names}), dict({k: -1 for k in names}), dict({k: 1 << 31 for k in names})]


VOX_RES = "res must be in 1..1024"
C_CHECKS = [
    ("gsr_dist2", dict(n=10, xyz=_P, scratch_alloc=_FN, scratch_user=None, dist2=_P, stream=None), [
        (_range("n"), _counts("n")),
        ("xyz, scratch_alloc and dist2 are required", [dict(xyz=None), dict(scratch_alloc=_NULL_FN), dict(dist2=None)]),
    ]),
    ("gsr_normal2rotation", dict(n=10, normals=_P, rot=_P, stream=None), [
        (_range("n"), _counts("n")),
        ("normals and rot are required", [dict(normals=None), dict(rot=None)]),
        ("rot must be 16-byte aligned", [dict(rot=_P + 4), dict(rot=_P + 8)]),
    ]),
    ("gsr_mesh_vertex_normals", dict(nv=10, verts=_P, nf=4, faces=_P, scratch_alloc=_FN, scratch_user=None,
                                     normals=_P, stream=None), [
        (_range("nv"), _counts("nv")),
        (_range("nf"), _counts("nf")),
        ("nf must be below 2^31 / 3", [dict(nf=0x7fffffff // 3 + 1), dict(nf=0x7fffffff)]),
        ("verts, faces, scratch_alloc and normals are required",
         [dict(verts=None), dict(faces=None), dict(scratch_alloc=_NULL_FN), dict(normals=None)]),
    ]),
    ("gsr_mesh_gaussians", dict(nf=4, n=3, verts=_P, faces=_P, vertex_normals=_P, colors=None, xyz=_P, rot=_P,
                                f_dc=_P, scale=_P, opacity=_P, stream=None), [
        (_range("nf"), _counts("nf")),
        ("n must be 1, 3, 4 or 6", [dict(n=0), dict(n=2), dict(n=5), dict(n=7), dict(n=-1)]),
        ("verts, faces, vertex_normals and every output are required",
         [dict(verts=None), dict(faces=None), dict(vertex_normals=None), dict(xyz=None), dict(rot=None),
          dict(f_dc=None), dict(scale=None), dict(opacity=None)]),
        ("rot must be 16-byte aligned", [dict(rot=_P + 4)]),
    ]),
    ("gsr_voxelize", dict(nv=10, verts=_P, nf=4, faces=_P, res=16, voxel_size=0.0625, alloc=_FN, column_user=None,
                          hit_user=None, sort_user=None, out_user=None, n_pairs=_P, stream=None), [
        (_range("nv"), _counts("nv")),
        (_range("nf"), _counts("nf")),
        (VOX_RES, [dict(res=0), dict(res=1025)]),
        ("voxel_size must be positive and finite",
         [dict(voxel_size=0.0), dict(voxel_size=-1.0), dict(voxel_size=math.nan), dict(voxel_size=math.inf)]),
        ("verts, faces, alloc and n_pairs are required",
         [dict(verts=None), dict(faces=None), dict(alloc=_NULL_FN), dict(n_pairs=None)]),
    ]),
    ("gsr_voxel_colors", dict(ncell=10, cells=_P, offsets=_P, tris=_P, res=16, voxel_size=0.0625, verts=_P, faces=_P,
                              colors=_P, rgb=_P, stream=None), [
        (_range("ncell"), _counts("ncell")),
        (VOX_RES, [dict(res=0), dict(res=1025)]),
        ("cells, offsets, tris, verts, faces, colors and rgb are required",
         [dict(cells=None), dict(offsets=None), dict(tris=None), dict(verts=None), dict(faces=None),
          dict(colors=None), dict(rgb=None)]),
    ]),
]


@pytest.mark.parametrize("entry,base,checks", C_CHECKS, ids=[c[0] for c in C_CHECKS])
def test_c_refusals_fire_in_order_before_any_work(entry, base, checks):
    """Each check returns -1 with its text, alone and together with the triggers of every later check."""
    fn = getattr(_lib.lib(), entry)
    for k, (err, variants) in enumerate(checks):
        later = {}
        for _, vs in reversed(checks[k + 1:]):
            later.update(vs[0])
        for v in variants:
            for over in (v, {**later, **v}):
                args = {**base, **over}
                assert fn(*args.values()) == -1, (entry, over)
                assert _lib.last_error() == f"{entry}: {err}", (entry, over, _lib.last_error())
