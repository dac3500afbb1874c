"""Point-cloud cleaning without a GPU: the float64 restatement (tests/clean_ref64.py) against hand-computed cases, the
checker against a seeded break of each rule, and every argument refusal of the Python functions and the C entries."""
import math

import numpy as np
import pytest
import torch

import clean_ref64 as C
from gaustudio_b200 import _lib, extract


def lattice(m=4, a=0.1):
    g = np.arange(-m, m + 1) * a
    X, Y, Z = np.meshgrid(g, g, g, indexing="ij")
    return np.c_[X.ravel(), Y.ravel(), Z.ravel()].astype(np.float32)


def test_cubic_lattice_interior_mean_distance():
    """The 50 nearest of an interior point: self, 6 at a, 12 at sqrt2 a, 8 at sqrt3 a, 6 at 2a, 17 of the 24 at sqrt5 a."""
    a = 0.25
    P = lattice(4, a)
    r = C.statistical64(P, 50)
    c = int(np.argmin(np.abs(P).sum(1)))
    want = a * (6 + 12 * math.sqrt(2) + 8 * math.sqrt(3) + 12 + 17 * math.sqrt(5)) / 50
    assert abs(r["avg"][c] - want) <= 1e-15
    assert r["keep"][c]


def test_lone_floater_is_dropped():
    x, n = C.surface("sphere", 2000)
    x = np.r_[x, [[40.0, 0.0, 0.0]]].astype(np.float32)
    r = C.statistical64(x, 50)
    assert not r["keep"][-1] and r["keep"][:-1].mean() > 0.9


@pytest.mark.parametrize("N", [0, 1, 2])
def test_tiny_clouds(N):
    x = np.random.default_rng(N).normal(size=(N, 3)).astype(np.float32)
    r = C.statistical64(x, 50)
    assert not r["keep"].any()  # N = 1: avg 0; N = 2: both avg equal the mean, and std 0 makes the test strict
    n = np.tile(np.float32([0, 0, 1]), (N, 1))
    assert not C.normal64(x, n)["keep"].any() if N < 2 else C.normal64(x, n)["keep"].all()


def test_fewer_points_than_k_and_coincident_points():
    x = np.random.default_rng(0).normal(size=(30, 3)).astype(np.float32)
    r = C.statistical64(x, 50)
    assert r["K"] == 30
    same = np.ones((10, 3), np.float32)
    assert not C.statistical64(same, 5)["keep"].any()  # avg 0 everywhere


def test_k_copies_of_one_point_are_dropped():
    x, _ = C.surface("plane", 500)
    x = np.r_[x, np.tile(np.float32([[0.3, 0.3, 0.2]]), (50, 1))]
    r = C.statistical64(x, 50)
    assert (r["avg"][-50:] == 0).all() and not r["keep"][-50:].any()


def test_236_plane_literal_drops_all_clamped_keeps_all():
    nv = torch.nn.functional.normalize(torch.tensor([[2.0, 3.0, 6.0]]), dim=1).numpy()[0]
    assert float((nv.astype(np.float64) ** 2).sum()) > 1.0
    g = np.random.default_rng(2).uniform(-1, 1, (800, 2))
    e1 = np.cross(nv, [1.0, 0, 0]); e1 /= np.linalg.norm(e1)
    e2 = np.cross(nv, e1)
    x = (g[:, :1] * e1 + g[:, 1:] * e2).astype(np.float32)
    n = np.tile(nv, (len(x), 1)).astype(np.float32)
    assert not C.normal64(x, n, literal=True)["keep"].any()
    assert C.normal64(x, n)["keep"].all()


def test_nan_normal_drops_its_neighbourhood():
    x, n = C.surface("plane", 1000)
    n[10] = np.nan
    r = C.normal64(x, n)
    assert not r["keep"][10]
    hit = (r["others"] == 10).any(1)
    assert hit.sum() > 0 and not r["keep"][hit].any()


# ---- the checker catches each seeded rule break ----
def _scene(seed=0):
    x, n = C.surface("torus", 1500, seed)
    x, n, _ = C.with_floaters(x, n, 0.03, far=1.5, seed=seed)
    return x, n


@pytest.mark.parametrize("fault", ["no_self", "population", "le", "no_pos"])
def test_checker_reports_pass1_faults(fault):
    x, _ = _scene()
    if fault == "le":  # a point exactly at the threshold: three points in a row, equally spaced
        x = np.float32([[0, 0, 0], [1, 0, 0], [2, 0, 0], [3, 0, 0]])
    if fault == "no_pos":
        x = np.r_[x, np.tile(np.float32([[0.9, 0.9, 0.9]]), (60, 1))]
    if fault == "population":  # Bessel's N - 1 matters on a small cloud: the first seed where a decision moves
        x = next(x for x in (np.random.default_rng(s).normal(size=(8, 3)).astype(np.float32) for s in range(1000))
                 if (C.statistical64(x, 3)["keep"] != C.statistical64(x, 3, fault=fault)["keep"]).any())
    k = 2 if fault == "le" else 3 if fault == "population" else 50
    ref = C.statistical64(x, k)
    bad = C.statistical64(x, k, fault=fault)
    if fault == "le":
        # every sum here is exact (avg = (0 + 1) / 2 = mean, std = 0): no rounding band around the threshold
        ref = dict(ref, bound_avg=ref["bound_avg"] * 0, bound_thr=0.0)
    with pytest.raises(C.CheckError):
        C.check_statistical(bad["avg"], bad["keep"], ref)
    assert C.check_statistical(ref["avg"], ref["keep"], ref) >= 0


@pytest.mark.parametrize("fault", ["idx0", "over_k", "fmin"])
def test_checker_reports_pass2_faults(fault):
    x, n = _scene(1)
    if fault == "fmin":
        n[::50] = np.nan
    ref = C.normal64(x, n)
    bad = C.normal64(x, n, fault=fault)
    with pytest.raises(C.CheckError):
        C.check_normal(bad["mean"], bad["keep"], ref, n)
    C.check_normal(ref["mean"], ref["keep"], ref, n)


def test_duplicates_and_ties_are_flagged_and_either_choice_accepted():
    x, n = C.surface("plane", 400, 3)
    x = np.r_[x, x[:5]]
    n = np.r_[n, -n[:5] * 0 + np.float32([1, 0, 0])]  # the copies point another way
    ref = C.normal64(x, n)
    assert ref["dup"].sum() == 10
    counts = C.check_normal(ref["mean"], ref["keep"], ref, n)
    assert counts["duplicates"] == 10
    g = lattice(3, 1.0)  # a lattice: cuts at the k-th neighbour are ties
    ref = C.normal64(g, np.tile(np.float32([0, 0, 1]), (len(g), 1)), k=10)
    assert ref["tie"].sum() > 0
    assert C.check_normal(ref["mean"], ref["keep"], ref, np.tile(np.float32([0, 0, 1]), (len(g), 1)), )["ties"] > 0


# ---- refusals ----
def _pts(n=10, dtype=torch.float32):
    return torch.rand(n, 3, dtype=dtype)


PY_REFUSALS = [
    (dict(xyz=[[0.0, 0.0, 0.0]]), "xyz must be a tensor"),
    (dict(xyz=_pts(dtype=torch.float64)), "must be float32"),
    (dict(normals=_pts(dtype=torch.float16)), "must be float32"),
    (dict(xyz=torch.rand(10, 4)), "must be [N,3]"),
    (dict(xyz=torch.rand(30)), "must be [N,3]"),
    (dict(normals=_pts(11)), "same shape"),
    (dict(k=0), "nb_neighbors must be"),
    (dict(k=65), "nb_neighbors must be"),
    (dict(k=20.0), "nb_neighbors must be"),
    (dict(k=True), "nb_neighbors must be"),
    (dict(ratio=0.0), "std_ratio must be"),
    (dict(ratio=-1.0), "std_ratio must be"),
    (dict(ratio=math.nan), "std_ratio must be"),
    (dict(ratio=math.inf), "std_ratio must be"),
    (dict(theta=math.nan), "angle_threshold must be"),
    (dict(theta=math.inf), "angle_threshold must be"),
    (dict(), "CUDA"),
]


def _call(fn, a):
    if fn == "remove_statistical_outlier":
        return extract.remove_statistical_outlier(a["xyz"], a["k"], a["ratio"])
    if fn == "remove_normal_outliers":
        return extract.remove_normal_outliers(a["xyz"], a["normals"], a["k"], a["theta"])
    return extract.clean_point_cloud(a["xyz"], _pts(len(a["xyz"]) if isinstance(a["xyz"], torch.Tensor) else 10),
                                     a["normals"], a["k"], a["ratio"])


@pytest.mark.parametrize("fn", ["remove_statistical_outlier", "remove_normal_outliers", "clean_point_cloud"])
@pytest.mark.parametrize("over,msg", PY_REFUSALS, ids=[m + str(i) for i, (_, m) in enumerate(PY_REFUSALS)])
def test_python_refusals_fire_before_device_work(fn, over, msg):
    uses = {"remove_statistical_outlier": ("xyz", "k", "ratio"), "remove_normal_outliers": ("xyz", "normals", "k", "theta"),
            "clean_point_cloud": ("xyz", "normals", "k", "ratio")}[fn]
    if any(key not in uses for key in over):
        pytest.skip("argument not taken by this function")
    if fn == "clean_point_cloud" and "xyz" in over and not isinstance(over["xyz"], torch.Tensor):
        msg = "rgb must be a tensor"
    args = dict(xyz=_pts(), normals=_pts(), k=20, ratio=2.0, theta=math.pi / 4)
    args.update(over)
    with pytest.raises(ValueError, match=msg.replace("[", r"\[").replace("]", r"\]")):
        _call(fn, args)


def test_clean_point_cloud_refuses_a_mismatched_rgb():
    with pytest.raises(ValueError, match="rgb"):
        extract.clean_point_cloud(_pts(), _pts(9), _pts())


_NULL_FN = _lib.ALLOC_FN()
_FN = _lib.ALLOC_FN(lambda u, n: 0)
_P = 1 << 20  # fake device address, never dereferenced: every call below is refused before any work
N_RANGE = "n must be in 1..2^31-1"
K_RANGE = "k must be in 1..64"
C_CHECKS = [
    ("gsr_clean_knn", dict(n=10, xyz=_P, k=5, scratch_alloc=_FN, scratch_user=None, index=_P, sq_dist=_P, stream=None), [
        (N_RANGE, [dict(n=0), dict(n=-1), dict(n=1 << 31)]),
        (K_RANGE, [dict(k=0), dict(k=65)]),
        ("xyz, scratch_alloc, index and sq_dist are required",
         [dict(xyz=None), dict(scratch_alloc=_NULL_FN), dict(index=None), dict(sq_dist=None)]),
    ]),
    ("gsr_clean_statistical", dict(n=10, xyz=_P, k=50, std_ratio=2.0, scratch_alloc=_FN, scratch_user=None,
                                   avg_dist=_P, stats=_P, keep=_P, stream=None), [
        (N_RANGE, [dict(n=0), dict(n=1 << 31)]),
        (K_RANGE, [dict(k=0), dict(k=-3), dict(k=65)]),
        ("std_ratio must be positive and finite",
         [dict(std_ratio=0.0), dict(std_ratio=-1.0), dict(std_ratio=math.nan), dict(std_ratio=math.inf)]),
        ("xyz, scratch_alloc, avg_dist, stats and keep are required",
         [dict(xyz=None), dict(scratch_alloc=_NULL_FN), dict(avg_dist=None), dict(stats=None), dict(keep=None)]),
    ]),
    ("gsr_clean_normal", dict(n=10, xyz=_P, normals=_P, k=20, angle_threshold=0.7, scratch_alloc=_FN,
                              scratch_user=None, mean_angle=_P, keep=_P, stream=None), [
        (N_RANGE, [dict(n=-5)]),
        (K_RANGE, [dict(k=100)]),
        ("angle_threshold must be finite",
         [dict(angle_threshold=math.nan), dict(angle_threshold=math.inf), dict(angle_threshold=-math.inf)]),
        ("xyz, normals, scratch_alloc, mean_angle and keep are required",
         [dict(xyz=None), dict(normals=None), dict(scratch_alloc=_NULL_FN), dict(mean_angle=None), dict(keep=None)]),
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
