"""CPU: the VisualHull and depth initializers' restatements (tests/hull_ref64.py) against the reference's own outputs
(tests/golden/hull_golden.npz, made by tests/golden/make_golden_hull.py), Camera's per-view fields and resizes, the
hull mesh restatement's topology, and every refusal before any device call."""
import math
import os

import numpy as np
import pytest
import torch

import hull_ref64 as R
import sap_ref64
from gaustudio_b200 import _lib, initializers
from gaustudio_b200.camera import Camera, look_at_camera, orbit_cameras
from gaustudio_b200.synthetic import GaussianPointCloud

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hull_golden.npz"))


def golden_cams():
    out = []
    for c in range(len(G["inside_size"])):
        W, H = (int(v) for v in G["inside_size"][c])
        fx, fy = G["inside_fov"][c]
        cam = Camera(R=G["inside_R"][c], T=G["inside_T"][c], FoVx=float(fx), FoVy=float(fy), image_width=W,
                     image_height=H)
        out.append((cam, W, H, G[f"inside_mask{c}"]))
    return out


@pytest.mark.parametrize("r,res", [(1.0, 2), (1.2, 128), (0.7371, 512), (3.3e-3, 97), (250.0, 129)])
def test_linspace_is_numpys(r, res):
    assert np.array_equal(R.linspace64(r, res), np.linspace(-r, r, res))


def test_grid_points_are_the_reference_meshgrid():
    r, res, t = 0.913, 9, np.array([0.25, -1.5, 3.125e-2])
    lin = np.linspace(-r, r, res)
    x, y, z = np.meshgrid(lin, lin, lin)  # mask.py:43-51
    ref = (np.stack([x.flatten(), y.flatten(), z.flatten()], axis=-1) - t).astype(np.float32)
    assert np.array_equal(R.grid_points(res, r, t).numpy(), ref)


def test_golden_projection_is_cameras():
    for c, (cam, W, H, _) in enumerate(golden_cams()):
        assert np.array_equal(cam.full_proj_transform.numpy(), G["inside_proj"][c])


@pytest.mark.parametrize("with_mask", [True, False])
def test_inside64_matches_reference_insideview(with_mask):
    x = torch.from_numpy(G["inside_points"])
    ref = G["inside_ref" if with_mask else "inside_nomask"]
    flagged_total = 0
    for c, (cam, W, H, m) in enumerate(golden_cams()):
        ins, flag = R.inside64(x, cam.full_proj_transform, W, H, m if with_mask else None)
        ins, flag = ins.numpy(), flag.numpy()
        bad = (ins != ref[c]) & ~flag
        assert not bad.any(), f"camera {c}: {np.flatnonzero(bad)[:10]}"
        flagged_total += int(flag.sum())
        # the torch restatement the GPU tests use is the reference's own computation
        got32 = R.inside_view32(x, cam.full_proj_transform, W, H, torch.from_numpy(m) if with_mask else None)
        assert np.array_equal(got32.numpy(), ref[c])
    # the bound flags the edge points of the 90-degree camera and a few pixel edges, not the scene
    assert flagged_total < 0.2 * x.shape[0]


def test_exact_ndc_edges_are_inside_and_behind_is_outside():
    cam, W, H, _ = golden_cams()[2]
    x = torch.from_numpy(G["inside_points"])
    ins, _ = R.inside64(x, cam.full_proj_transform, W, H)
    edge = slice(3000, 3000 + 4 * 64)
    assert ins[edge].all() and G["inside_nomask"][2][edge].all()
    behind = slice(3000 + 4 * 64, 3000 + 6 * 64)
    assert not ins[behind].any() and not G["inside_nomask"][2][behind].any()


def test_carve64_matches_carve32_outside_flags():
    cams = orbit_cameras(6, 4.0, 20.0, 64, 48, 0.9, 0.7)
    rng = np.random.default_rng(0)
    masks = [(rng.uniform(size=(48, 64)) < 0.8) for _ in cams]
    specs = [(c.full_proj_transform, 64, 48, m) for c, m in zip(cams, masks)]
    x = R.grid_points(24, 1.3, np.zeros(3))
    occ, flag = R.carve64(x, specs)
    ref = R.carve32(x, specs)
    assert not ((occ != ref) & ~flag).any()
    assert flag.float().mean() < 0.1


@pytest.mark.parametrize("tag", ["s4", "r2011"])
def test_camera_downsample_is_the_references(tag):
    H, W = G["rs_image"].shape[:2]
    cam = Camera(R=np.eye(3), T=np.zeros(3), FoVx=1.0, FoVy=0.8, image_width=W, image_height=H,
                 image=torch.from_numpy(G["rs_image"]), mask=torch.from_numpy(G["rs_mask"]),
                 depth=torch.from_numpy(G["rs_depth"]))
    out = cam.downsample_scale(4) if tag == "s4" else cam.downsample((20, 11))
    assert out is cam
    for k in ("image", "mask", "depth"):
        got = getattr(cam, k).numpy()
        assert got.dtype == G[f"rs_{tag}_{k}"].dtype and np.array_equal(got, G[f"rs_{tag}_{k}"]), k
    assert [cam.image_width, cam.image_height] == list(G[f"rs_{tag}_size"])


def test_camera_fields_default_and_focal_lengths():
    cam = Camera(R=np.eye(3), T=np.zeros(3), FoVx=1.0, FoVy=0.8, image_width=40, image_height=30)
    assert cam.image is None and cam.mask is None and cam.depth is None
    assert cam.fx.dtype == torch.float32 and cam.fx.dim() == 0 and float(cam.fx) == float(cam.intrinsics[0, 0])
    assert float(cam.fy) == float(cam.intrinsics[1, 1])
    with pytest.raises(ValueError, match="Depth is not available"):
        cam.depth2point()


def golden_depth_views():
    return [(G[f"dc_xyz{i}"], G[f"dc_image{i}"], G[f"dc_depth{i}"], *G[f"dc_f{i}"]) for i in range(2)]


def test_depth_chain_is_the_references():
    d = R.depth_chain(golden_depth_views())
    assert np.array_equal(d["points16"], G["dc_points16"])
    assert np.array_equal(d["colors"], G["dc_colors"])
    assert np.array_equal(d["scales16"], G["dc_scales16"])
    assert np.array_equal(d["xyz"], G["dc_model_xyz"])
    assert np.array_equal(d["rgb"], G["dc_model_rgb"])
    assert np.array_equal(d["log_scale"], G["dc_model_log_scale"])  # -inf where the depth is 0
    assert np.isneginf(d["log_scale"]).any()
    assert np.array_equal(d["opacity"], G["dc_model_opacity"])


def sphere_occ(res, r, t, rad, centre):
    x = R.grid_points(res, r, t).double().numpy()
    return (np.linalg.norm(x - centre, axis=1) <= rad).reshape(res, res, res)


@pytest.mark.parametrize("threshold", [0.25, 0.5, 0.75])
def test_hull_mesh64_is_closed_outward_and_on_the_edges(threshold):
    res, r, t = 20, 1.0, np.array([0.1, -0.05, 0.2])
    occ = sphere_occ(res, r, t, 0.6, np.array([-0.1, 0.05, -0.2]))
    v, f, w = R.hull_mesh64(occ, threshold, r, t)
    closed, euler = sap_ref64.edge_manifold(f)
    assert closed and euler == 2
    assert R.signed_volume(w, f) > 0
    crossing = sum(int((occ[tuple(slice(0, res - 1) if b == a else slice(None) for b in range(3))] !=
                        occ[tuple(slice(1, res) if b == a else slice(None) for b in range(3))]).sum())
                   for a in range(3))
    assert len(v) == crossing
    # each vertex lies on its grid edge, `threshold` of the way from the empty node
    q = np.stack([(w[:, 1] + t[1] + r), (w[:, 0] + t[0] + r), (w[:, 2] + t[2] + r)], 1) / (2 * r) * (res - 1)
    frac = q - np.floor(q + 1e-9)
    on_edge = np.abs(frac) < 1e-9
    assert (on_edge.sum(1) == 2).all()
    c = np.floor(q + 1e-9).astype(int)
    f_at = frac[~on_edge]
    start_filled = occ[c[:, 0], c[:, 1], c[:, 2]]
    assert np.allclose(f_at, np.where(start_filled, 1 - threshold, threshold), atol=1e-9)


# ---- refusals: every one before any device call ----
@pytest.fixture
def no_device(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("device call before the refusal")
    monkeypatch.setattr(initializers, "call", boom)


@pytest.mark.parametrize("cfg", [{"resolution": 1}, {"resolution": 513}, {"resolution": 64.0}, {"resolution": True},
                                 {"threshold": 0.0}, {"threshold": 1.0}, {"threshold": float("nan")},
                                 {"radius_scale": float("inf")}])
def test_visual_hull_config_refusals(cfg, tmp_path, no_device):
    with pytest.raises(ValueError):
        initializers.make({"name": "VisualHull", "workspace_dir": str(tmp_path), **cfg})


def test_visual_hull_refuses_a_zero_radius(tmp_path, no_device):
    init = initializers.make({"name": "VisualHull", "workspace_dir": str(tmp_path)})
    model = GaussianPointCloud.empty(device="cpu")
    with pytest.raises(ValueError, match="radius"):
        init(model, [look_at_camera((3, 0, 0), (0, 0, 0), 40, 30, 0.9, 0.7)])  # one camera: min_radius 0
    negative = initializers.make({"name": "VisualHull", "workspace_dir": str(tmp_path), "radius_scale": -1.0})
    with pytest.raises(ValueError, match="radius"):
        negative(model, orbit_cameras(4, 3.0, 0.0, 40, 30, 0.9, 0.7))
    with pytest.raises(ValueError, match="no cameras"):
        init(model, [])
    assert not os.path.exists(tmp_path / "visual_hull.ply")


def test_visual_hull_refuses_a_mask_of_another_shape(tmp_path, no_device):
    cams = orbit_cameras(4, 3.0, 10.0, 40, 30, 0.9, 0.7)
    for c in cams:
        c.mask = torch.ones(30, 40)
    cams[2].mask = torch.ones(40, 30)
    init = initializers.make({"name": "VisualHull", "workspace_dir": str(tmp_path)})
    with pytest.raises(ValueError, match="mask"):
        init(GaussianPointCloud.empty(device="cpu"), cams)


def test_depth_refusals(tmp_path, no_device):
    init = initializers.make({"name": "depth", "workspace_dir": str(tmp_path)})
    model = GaussianPointCloud.empty(device="cpu")
    cams = orbit_cameras(2, 3.0, 10.0, 40, 32, 0.9, 0.7)
    with pytest.raises(ValueError, match="no camera has a depth"):
        init(model, cams)
    cams[0].depth = torch.ones(32, 40)
    with pytest.raises(ValueError, match="of the same size"):
        init(model, cams)  # no image
    cams[0].image = torch.rand(32, 44, 3)
    with pytest.raises(ValueError, match="of the same size"):
        init(model, cams)
    cams[0].image = torch.rand(32, 40, 3)
    with pytest.raises(ValueError, match="CUDA"):
        init(model, cams)  # a CPU model, after the views passed
    assert cams[0].image_width == 40 and tuple(cams[0].depth.shape) == (32, 40)  # the caller's camera is untouched
    assert not os.path.exists(tmp_path / "fused.ply")


# ---- refusals of the C entries: each check returns -1 with its text, before any device work ----
_NULL_FN = _lib.ALLOC_FN()
_FN = _lib.ALLOC_FN(lambda u, n: 0)
_P = 1 << 20  # fake device address, never dereferenced: every call below is refused before any work
RES = "res must be in 2..512"
RADIUS = "radius must be positive and finite"
TRANSLATE = "translate must be finite"
C_CHECKS = [
    ("gsr_hull_carve", dict(res=32, radius=1.0, tx=0.0, ty=0.0, tz=0.0, n_cams=2, proj=_P, views=_P, masks=_P,
                            occ=_P, stream=None), [
        (RES, [dict(res=1), dict(res=513), dict(res=-4)]),
        (RADIUS, [dict(radius=0.0), dict(radius=-1.0), dict(radius=math.nan), dict(radius=math.inf),
                  dict(radius=1e300)]),
        (TRANSLATE, [dict(tx=math.nan), dict(ty=math.inf), dict(tz=-math.inf)]),
        ("n_cams must be >= 0", [dict(n_cams=-1)]),
        ("occ, proj and views are required", [dict(occ=None), dict(proj=None), dict(views=None)]),
    ]),
    ("gsr_hull_marching_cubes", dict(res=32, occ=_P, threshold=0.5, radius=1.0, tx=0.0, ty=0.0, tz=0.0,
                                     scratch_alloc=_FN, scratch_user=None, vertex_alloc=_FN, vertex_user=None,
                                     face_alloc=_FN, face_user=None, n_faces=_P, stream=None), [
        (RES, [dict(res=1), dict(res=513)]),
        ("threshold must be in (0, 1)", [dict(threshold=0.0), dict(threshold=1.0), dict(threshold=math.nan)]),
        (RADIUS, [dict(radius=0.0), dict(radius=math.inf)]),
        (TRANSLATE, [dict(tx=math.inf), dict(ty=math.nan), dict(tz=math.nan)]),
        ("occ is required", [dict(occ=None)]),
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
