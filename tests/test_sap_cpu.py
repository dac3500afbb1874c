"""Shape-as-Points meshing without a GPU: the float64 restatement (tests/sap_ref64.py) against what the reference's own
DPSR computed (tests/golden/sap_golden.npz, tests/golden/make_golden_sap.py), the geometry it produces, the splat's
conservation, wrap and on-node rules, and every argument refusal of extract.mesh_sap / extract.dpsr and of the C entries."""
import math
import os

import numpy as np
import pytest
import torch

import sap_ref64 as S
from gaustudio_b200 import _lib, extract

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sap_golden.npz")
U = S.U32


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


def _terms_per_node(p, res):
    i0, _ = S.axis_weights(p, res)
    cnt = np.zeros(res ** 3)
    for ox, oy, oz in S.corners():
        np.add.at(cnt, (((i0[:, 0] + ox) % res) * res + (i0[:, 1] + oy) % res) * res + (i0[:, 2] + oz) % res, 1)
    return cnt.reshape(res, res, res)


@pytest.mark.parametrize("shape", list(S.SHAPES))
@pytest.mark.parametrize("res", [32, 64])
def test_restatement_matches_the_reference_grids(gold, shape, res):
    """The reference splats and solves in float32: per node its splat differs from float64 by at most
    (8 + k) u sum|terms| (8 roundings per weighted term, k - 1 in a k-term sum), and its DPSR output by the
    float32 bound of sap_ref64.psi_bound (that bound covers the argument of the tanh)."""
    p, n = gold[f"{shape}_p"], gold[f"{shape}_normals"]
    ref = S.dpsr64(p.astype(np.float64), n, res)
    r = 1 if res == 32 else 2  # the golden file keeps the res-64 splat on every 2nd node
    bound = ((8.0 + _terms_per_node(p, res)) * U * ref["mag"])[::r, ::r, ::r]
    err = np.abs(ref["grid"][:, ::r, ::r, ::r] - gold[f"{shape}_raster_{res}"])
    assert (err <= bound[None] + 1e-30).all(), (err / (bound[None] + 1e-30)).max()
    phi = gold[f"{shape}_phi_{res}"]
    k = res // 16  # the golden file keeps phi on a 16^3 subgrid
    mine = ref["scaled"][::k, ::k, ::k]
    tol = S.psi_bound(ref, res)
    assert np.abs(mine - phi).max() <= tol, (np.abs(mine - phi).max(), tol)


@pytest.mark.parametrize("r", [0.3, 0.5])
def test_sphere_zero_level_lies_at_its_radius(r):
    centre = np.array([0.1, -0.2, 0.3])
    xyz, n = S.sphere(4000, r=r, centre=centre)
    v, f, ref, c, s = S.mesh64(xyz, n, 64)
    voxel = 2.0 * s / 64
    dist = np.linalg.norm(v - centre, axis=1)
    assert np.abs(dist - r).max() < voxel, (np.abs(dist - r).max(), voxel)
    closed, euler = S.edge_manifold(f)
    assert closed and euler == 2
    nrm = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    assert (np.einsum("ij,ij->i", nrm, v[f].mean(1) - centre) > 0).all()  # outward
    assert ref["psi"][0, 0, 0] > 0 > ref["psi"][tuple(np.floor(((centre - c) / s + 1) / 2 * 64).astype(int))]


@pytest.mark.parametrize("shape", list(S.SHAPES))
def test_splat_conserves_the_normal_sum(gold, shape):
    p, n = gold[f"{shape}_p"].astype(np.float64), gold[f"{shape}_normals"].astype(np.float64)
    for res in (32, 64):
        grid, _ = S.splat64(p, n, res)
        np.testing.assert_allclose(grid.reshape(3, -1).sum(1), n.sum(0), rtol=0, atol=1e-9 * np.abs(n).sum())
    ref = gold[f"{shape}_raster_32"].astype(np.float64)  # the one golden splat kept whole
    np.testing.assert_allclose(ref.reshape(3, -1).sum(1), n.sum(0), rtol=0, atol=1e-5 * np.abs(n).sum())


def test_splat_wraps_periodically_and_gives_on_node_points_to_i0():
    res = 8
    n = np.array([[1.0, 2.0, 3.0]])
    # between node 7 and node 8 == 0 on x: a quarter of the way
    g, _ = S.splat64(np.array([[7.25 / res, 2.0 / res, 5.0 / res]]), n, res)
    assert np.isclose(g[0, 7, 2, 5], 0.75) and np.isclose(g[0, 0, 2, 5], 0.25)
    assert np.count_nonzero(g[0]) == 2 and np.allclose(g[:, 0, 2, 5], 0.25 * n[0])
    # exact multiples of 1/res on every axis: all of the weight on the node itself
    g, _ = S.splat64(np.array([[3.0 / res, 0.0, 7.0 / res]]), n, res)
    assert np.count_nonzero(g[1]) == 1 and g[1, 3, 0, 7] == 2.0
    # the interpolation uses the same weights and the same wrap
    phi = np.random.default_rng(0).normal(size=(res, res, res))
    q = np.array([[7.5 / res, 0.25 / res, 6.0 / res]])
    want = 0.5 * (0.75 * phi[7, 0, 6] + 0.25 * phi[7, 1, 6]) + 0.5 * (0.75 * phi[0, 0, 6] + 0.25 * phi[0, 1, 6])
    assert np.isclose(S.interp64(phi, q)[0], want)


def test_marching_cubes_restatement_faces_point_to_positive_psi():
    r = 12
    x = np.arange(r)
    X, Y, Z = np.meshgrid(x, x, x, indexing="ij")
    psi = np.sqrt((X - 5.3) ** 2 + (Y - 5.6) ** 2 + (Z - 5.1) ** 2) - 3.0  # negative inside a ball of radius 3
    v, f = S.marching_cubes64(psi)
    closed, euler = S.edge_manifold(f)
    assert closed and euler == 2 and len(np.unique(f)) == len(v)
    assert np.abs(S.trilinear(psi, v)).max() < 1e-12
    nrm = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    assert (np.einsum("ij,ij->i", nrm, v[f].mean(1) - [5.3, 5.6, 5.1]) > 0).all()


# ---- refusals ----
def _pts(n=10, dtype=torch.float32):
    return torch.rand(n, 3, dtype=dtype)


PY_REFUSALS = [
    (dict(xyz=[[0.0, 0.0, 0.0]]), "must be a tensor"),
    (dict(xyz=_pts(dtype=torch.float64)), "must be float32"),
    (dict(normals=_pts(dtype=torch.float16)), "must be float32"),
    (dict(xyz=torch.rand(10, 4)), "must be [N,3]"),
    (dict(xyz=torch.rand(30)), "must be [N,3]"),
    (dict(normals=_pts(11)), "same shape"),
    (dict(xyz=_pts(0), normals=_pts(0)), "at least one point"),
    (dict(res=1), "res must be"),
    (dict(res=513), "res must be"),
    (dict(res=64.0), "res must be"),
    (dict(res=True), "res must be"),
    (dict(sig=0.0), "sig must be"),
    (dict(sig=-1), "sig must be"),
    (dict(sig=math.nan), "sig must be"),
    (dict(sig=math.inf), "sig must be"),
    (dict(), "CUDA"),
]


@pytest.mark.parametrize("fn", ["mesh_sap", "dpsr"])
@pytest.mark.parametrize("over,msg", PY_REFUSALS, ids=[m + str(i) for i, (_, m) in enumerate(PY_REFUSALS)])
def test_python_refusals_fire_before_device_work(fn, over, msg):
    args = dict(xyz=_pts(), normals=_pts(), res=32, sig=2)
    args.update(over)
    with pytest.raises(ValueError, match=msg.replace("[", r"\[").replace("]", r"\]")):
        getattr(extract, fn)(args["xyz"], args["normals"], res=args["res"], sig=args["sig"])


_NULL_FN = _lib.ALLOC_FN()
_FN = _lib.ALLOC_FN(lambda u, n: 0)
_P = 1 << 20  # fake device address, never dereferenced: every call below is refused before any work
N_RANGE = "n must be in 1..2^31-1"
RES = "res must be in 2..512"
C_CHECKS = [
    ("gsr_sap_normalize", dict(n=10, xyz=_P, scratch_alloc=_FN, scratch_user=None, points01=_P, transform=_P,
                               stream=None), [
        (N_RANGE, [dict(n=0), dict(n=-1), dict(n=1 << 31)]),
        ("xyz, points01, transform and scratch_alloc are required",
         [dict(xyz=None), dict(points01=None), dict(transform=None), dict(scratch_alloc=_NULL_FN)]),
    ]),
    ("gsr_sap_splat", dict(n=10, points01=_P, normals=_P, res=32, scratch_alloc=_FN, scratch_user=None, grid=_P,
                           stream=None), [
        (N_RANGE, [dict(n=0)]),
        (RES, [dict(res=1), dict(res=513)]),
        ("points01, normals, grid and scratch_alloc are required",
         [dict(points01=None), dict(normals=None), dict(grid=None), dict(scratch_alloc=_NULL_FN)]),
    ]),
    ("gsr_sap_spectral", dict(res=32, sig=2.0, spectrum=_P, phi_hat=_P, stream=None), [
        (RES, [dict(res=0)]),
        ("sig must be positive and finite", [dict(sig=0.0), dict(sig=math.nan), dict(sig=math.inf)]),
        ("spectrum and phi_hat are required", [dict(spectrum=None), dict(phi_hat=None)]),
    ]),
    ("gsr_sap_shift_scale", dict(n=10, points01=_P, res=32, phi=_P, scratch_alloc=_FN, scratch_user=None, psi=_P,
                                 stream=None), [
        (N_RANGE, [dict(n=-5)]),
        (RES, [dict(res=1000)]),
        ("points01, phi, psi and scratch_alloc are required",
         [dict(points01=None), dict(phi=None), dict(psi=None), dict(scratch_alloc=_NULL_FN)]),
    ]),
    ("gsr_sap_marching_cubes", dict(res=32, psi=_P, transform=_P, scratch_alloc=_FN, scratch_user=None,
                                    vertex_alloc=_FN, vertex_user=None, face_alloc=_FN, face_user=None, n_faces=_P,
                                    stream=None), [
        (RES, [dict(res=1)]),
        ("psi and transform are required", [dict(psi=None), dict(transform=None)]),
        ("allocators and n_faces are required",
         [dict(scratch_alloc=_NULL_FN), dict(vertex_alloc=_NULL_FN), dict(face_alloc=_NULL_FN), dict(n_faces=None)]),
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
