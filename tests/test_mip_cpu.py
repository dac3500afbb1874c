"""The Mip-Splatting path without a GPU: the float64 references of tests/mip_ref64.py against finite differences, the
vanilla reference and a per-camera loop; the MipPointCloud model, its PLY round trip, the renderer's configuration
surface and the argument checks of the new C entry points."""
import math

import numpy as np
import pytest
import torch

import mip_ref64 as MR
import proj_ref64 as R
from test_abi import _call, _Off

F64 = torch.float64
W, H = 64, 48


def _scene(P, seed, collapse=()):
    """Un-fused float64 inputs in front of a camera; the rows in `collapse` get scales of 1e-7 (their cov2D collapses)."""
    from gaustudio_b200.camera import look_at_camera
    rng = np.random.RandomState(seed)
    fov = math.radians(50.0)
    cam = look_at_camera((2.2, 1.4, 1.6), (0, 0, 0), W, H, 2 * math.atan(math.tan(fov / 2) * W / H), fov)
    means = 0.4 * rng.randn(P, 3)
    s = 0.05 * np.exp(0.3 * rng.randn(P, 3))
    s[list(collapse)] = 1e-7
    q = rng.randn(P, 4)
    p = dict(means3D=means, shs=0.5 * rng.randn(P, 16, 3), opacities=0.1 + 0.8 * rng.rand(P, 1), scales=s, rotations=q)
    p = {k: torch.tensor(v, dtype=F64) for k, v in p.items()}
    Dcam = R.camera(cam.world_view_transform, cam.full_proj_transform, cam.camera_center, math.tan(cam.FoVx * 0.5),
                    math.tan(cam.FoVy * 0.5), W, H, 3, 1.0)
    return p, Dcam


def _loss(p, cam, k, up):
    s = MR.mip_state(R._params(p, False), cam, k)
    return ((up["mean2D"][:, :2] * s["ndc"]).sum() + (up["conic"] * s["conic"] * torch.tensor([1.0, 2.0, 1.0], dtype=F64)).sum()
            + (up["color"] * s["rgb"]).sum() + (up["depth"] * s["depth"]).sum() + (up["opacity"] * s["opacity"]).sum())


@pytest.mark.parametrize("k", [0.0, 0.1, 0.3, 2.0])
def test_vjp_matches_central_differences(k):
    """Every input's gradient against central differences of the float64 forward.  Rows 0 and 1 are collapsed: det0
    clamps for every k, det1 too at k = 0.  The conic upstream is 0 on rows with det(cov') < 1, where the reference's
    regularised conic backward (1 / (det^2 + 1e-7)) is not the exact derivative."""
    P = 10
    p, cam = _scene(P, 3 + int(10 * k), collapse=(0, 1))
    f = MR.forward(p, cam, k)
    assert (f["coef"][:2] == 0).all() and (f["coef"][2:] > 0).all()
    assert (f["det0"][:2] <= MR.EPS6).all()
    if k == 0.0:
        assert (f["det1"][:2] <= MR.EPS6).all()
    g = torch.Generator().manual_seed(1)
    a, b, c = f["cov2D"].unbind(1)
    well = ((a * c - b * b) >= 1.0)[:, None]
    up = dict(mean2D=torch.randn(P, 3, generator=g, dtype=F64), conic=torch.randn(P, 3, generator=g, dtype=F64) * well,
              color=torch.randn(P, 3, generator=g, dtype=F64), depth=torch.randn(P, generator=g, dtype=F64),
              opacity=torch.randn(P, generator=g, dtype=F64))
    radii = f["radius"].numpy()
    assert (radii > 0).all()
    ref = MR.vjp(p, cam, k, up, radii, f["clamped"].numpy())
    names = dict(means3D="means3D", shs="shs", opacities="opacity", scales="scales", rotations="rotations")
    for key, out in names.items():
        x = p[key]
        fd = torch.zeros_like(x)
        flat = x.reshape(-1)
        for i in range(flat.numel()):
            h = 1e-6 * max(1.0, abs(float(flat[i])))
            for sgn in (1, -1):
                q = {kk: v.clone() for kk, v in p.items()}
                q[key].reshape(-1)[i] += sgn * h
                fd.reshape(-1)[i] += sgn * float(_loss(q, cam, k, up)) / (2 * h)
        got = ref[out]
        if key == "shs":  # only the (D+1)^2 coefficients the forward reads move the loss
            got = got[:, :16]
        got = got.reshape(fd.shape)
        err = (got - fd).abs().max()
        assert err <= 1e-5 * max(1.0, float(fd.abs().max())), (key, float(err), float(fd.abs().max()))
    assert (ref["opacity"][:2] == 0).all()


def test_k03_matches_the_vanilla_reference():
    """At kernel_size 0.3, cov' is the vanilla 0.3-dilated cov2D: the same means2D, conic, radius and depth, and an
    opacity of o coef."""
    p, cam = _scene(200, 9, collapse=(5, 6, 7))
    f = MR.forward(p, cam, 0.3)
    v = R.forward(p, cam)
    for key in ("means2D", "conic", "depth", "rgb"):
        assert torch.allclose(f[key], v[key], rtol=1e-12, atol=1e-12), key
    assert torch.equal(f["radius"], v["radius"])
    assert torch.allclose(f["opacity"], p["opacities"].reshape(-1) * f["coef"], rtol=1e-15, atol=0)
    assert (f["coef"][5:8] == 0).all() and (f["coef"] <= 1).all()


def _loop_filter(xyz, cams):
    """A direct per-camera numpy loop written from the definition (include/gsr.h, gsr_mip_filter3d)."""
    d = np.full(len(xyz), 100000.0)
    seen = np.zeros(len(xyz), bool)
    fmax = 0.0
    for c in cams:
        fx = c.image_width / (2 * math.tan(c.FoVx / 2))
        fy = c.image_height / (2 * math.tan(c.FoVy / 2))
        p = xyz @ np.asarray(c.R) + np.asarray(c.T)
        z = np.maximum(p[:, 2], 0.001)
        u = p[:, 0] / z * fx + c.image_width / 2
        v = p[:, 1] / z * fy + c.image_height / 2
        ok = (p[:, 2] > 0.2) & (u >= -0.15 * c.image_width) & (u <= 1.15 * c.image_width) & \
             (v >= -0.15 * c.image_height) & (v <= 1.15 * c.image_height)
        d[ok] = np.minimum(d[ok], p[ok, 2])
        seen |= ok
        fmax = max(fmax, fx)
    if not seen.any():
        raise ValueError("nothing seen")
    d[~seen] = d[seen].max()
    return d / fmax * math.sqrt(0.2), seen


def test_filter3d_oracle_matches_a_per_camera_loop():
    from gaustudio_b200.camera import look_at_camera, orbit_cameras
    rng = np.random.RandomState(0)
    xyz = rng.randn(3000, 3)
    xyz[:5] = [[2e5, 0, 0], [2.5e5, 10, 0], [0, 0, 40], [0, 0, -40], [30, 30, 30]]
    cams = orbit_cameras(7, 3.0, 20.0, 64, 48, 0.8, 0.6) + [look_at_camera((-5, 0, 0), (0, 0, 0), 320, 240, 0.4, 0.3)]
    ref, seen = MR.filter3d(xyz, MR.camera_records(cams))
    loop, seen2 = _loop_filter(xyz, cams)
    assert np.array_equal(seen, seen2)
    assert np.allclose(ref, loop, rtol=1e-14, atol=0)
    fmax = max(c.image_width / (2 * math.tan(c.FoVx / 2)) for c in cams)
    assert seen[0] and seen[1] and ref[0] == ref[1] == 100000.0 / fmax * math.sqrt(0.2)  # the cap
    assert (~seen).sum() > 0 and np.all(ref[~seen] == ref[seen].max())                  # the fill
    with pytest.raises(ValueError):
        MR.filter3d(np.array([[0.0, 0.0, 1e3]]) + 1e7, MR.camera_records(cams))
    with pytest.raises(ValueError):
        _loop_filter(np.array([[0.0, 0.0, 1e3]]) + 1e7, cams)


def _mip_model(P=50, seed=0):
    from gaustudio_b200.mip import MipPointCloud
    g = torch.Generator().manual_seed(seed)
    m = MipPointCloud(torch.randn(P, 3, generator=g), -3 + 0.5 * torch.randn(P, 3, generator=g),
                      torch.randn(P, 4, generator=g), torch.randn(P, 1, generator=g), torch.randn(P, 1, 3, generator=g),
                      0.1 * torch.randn(P, 15, 3, generator=g), filter_3D=0.02 * torch.rand(P, 1, generator=g))
    return m


def test_mip_point_cloud_properties_match_numpy():
    m = _mip_model()
    s = np.exp(m._scale.numpy().astype(np.float64))
    f = m.filter_3D.numpy().astype(np.float64)
    o = 1 / (1 + np.exp(-m._opacity.numpy().astype(np.float64)))
    sf = np.sqrt(s ** 2 + f ** 2)
    assert np.allclose(m.get_scaling_with_3D_filter.numpy(), sf, rtol=1e-6)
    coef = np.sqrt(np.prod(s ** 2, 1) / np.prod(s ** 2 + f ** 2, 1))
    assert np.allclose(m.get_opacity_with_3D_filter.numpy(), o * coef[:, None], rtol=1e-5)
    q = m._rot.numpy().astype(np.float64)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    import scenes
    Rm = scenes.quat_to_mat(q)
    L = Rm * (1.7 * sf)[:, None, :]
    S = L @ L.transpose(0, 2, 1)
    packed = np.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], 1)
    assert np.allclose(m.get_covariance(1.7).numpy(), packed, rtol=1e-5, atol=1e-6 * np.abs(packed).max())
    assert not m.filter_3D.requires_grad
    assert m.filter_3D.shape == (50, 1)


def test_ply_round_trip_keeps_filter_3d(tmp_path):
    from gaustudio_b200 import io
    from gaustudio_b200.mip import MipPointCloud
    from gaustudio_b200.synthetic import GaussianPointCloud
    m = _mip_model()
    path = str(tmp_path / "m.ply")
    io.export_ply(m, path)
    back = io.load_ply(path)
    assert isinstance(back, MipPointCloud)
    assert torch.equal(back.filter_3D, m.filter_3D)
    for k in ("_xyz", "_scale", "_rot", "_opacity"):
        assert torch.equal(getattr(back, k), getattr(m, k).reshape(getattr(back, k).shape)), k
    assert io.read_ply_vertices(path).dtype.names[-1] == "filter_3D"
    # a PLY without the property loads as before, and writes no filter_3D
    plain = GaussianPointCloud(m._xyz, m._scale, m._rot, m._opacity, m._f_dc, m._f_rest)
    p2 = str(tmp_path / "plain.ply")
    io.export_ply(plain, p2)
    back2 = io.load_ply(p2)
    assert type(back2) is GaussianPointCloud and not hasattr(back2, "filter_3D")
    assert "filter_3D" not in io.read_ply_vertices(p2).dtype.names


def test_mip_renderer_config_surface():
    from gaustudio_b200 import renderers
    r = renderers.make("mip_renderer")
    assert r.kernel_size == 0.3 and r.scaling_modifier == 1.0 and not r.white_background
    assert not r.convert_SHs_python and not r.compute_cov3D_python and not r.debug
    assert r.bg_color.device.type == "cpu" and r.bg_color.tolist() == [0.0, 0.0, 0.0]
    conf = {"name": "mip_renderer", "kernel_size": 0.1, "scaling_modifier": 0.5, "white_background": True,
            "convert_SHs_python": True, "compute_cov3D_python": True, "debug": True}
    r = renderers.make(conf)
    assert (r.kernel_size, r.scaling_modifier, r.bg_color.tolist()) == (0.1, 0.5, [1.0, 1.0, 1.0])
    assert r.convert_SHs_python and r.compute_cov3D_python and r.debug
    for bad in (-0.1, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            renderers.make({"name": "mip_renderer", "kernel_size": bad})


def test_model_without_filter_is_refused_before_any_device_work():
    from gaustudio_b200 import renderers
    from gaustudio_b200.camera import look_at_camera
    from gaustudio_b200.mip import MipPointCloud
    from gaustudio_b200.synthetic import make_scene
    cam = look_at_camera((3, 0, 0), (0, 0, 0), 32, 32, 0.8, 0.8)
    r = renderers.make("mip_renderer")
    for model in (make_scene(20, 1.0, 0.01, 0), MipPointCloud.from_model(make_scene(20, 1.0, 0.01, 0))):
        with pytest.raises(ValueError, match="compute_3D_filter"):
            r.render(cam, model)  # CPU tensors: any device work would fail differently


def test_mip_settings_fields():
    from gaustudio_b200 import mip_rasterizer
    assert mip_rasterizer.GaussianRasterizationSettings._fields == (
        "image_height", "image_width", "tanfovx", "tanfovy", "kernel_size", "bg", "scale_modifier", "viewmatrix",
        "projmatrix", "sh_degree", "campos", "prefiltered", "debug")


KS = "kernel_size must be finite and >= 0"


@pytest.mark.parametrize("entry,extra,err", [
    ("gsr_forward_mip", {}, "gsr_forward_mip: " + KS),
    ("gsr_backward_mip", {}, "gsr_backward_mip: " + KS),
    ("gsr_debug_projection_backward_mip", {}, "gsr_debug_projection_backward_mip: " + KS)])
def test_mip_entry_points_refuse_bad_arguments_before_any_work(entry, extra, err):
    from gaustudio_b200 import _lib
    for k in (-0.1, float("nan"), float("inf"), -float("inf")):
        assert _call(entry, kernel_size=k, **extra) == -1
        assert _lib.last_error() == err
    if entry != "gsr_forward_mip":
        assert _call(entry, kernel_size=0.3, opacities=None) == -1
        assert _lib.last_error() == f"{entry}: opacities are required"
    # the checks of the entry point it extends follow
    if entry == "gsr_forward_mip":
        assert _call(entry, kernel_size=0.3, P=0) == -1
        assert _lib.last_error() == "gsr_forward: P, width and height must be positive"
        assert _call(entry, kernel_size=0.0, rotations=_Off(4)) == -1
        assert _lib.last_error() == "gsr_forward: rotations must be 16-byte aligned"
        assert _call(entry, kernel_size=0.3) == -1
        assert _lib.last_error() == "gsr_forward: scratch allocation failed"
    elif entry == "gsr_backward_mip":
        assert _call(entry, kernel_size=0.3, geom_buffer=None) == -1
        assert _lib.last_error() == "gsr_backward: missing state buffers"
    else:
        assert _call(entry, kernel_size=0.3, accum=None) == -1
        assert _lib.last_error() == "gsr_debug_projection_backward_mip: accum is required"


def test_filter3d_entry_point_checks():
    from gaustudio_b200 import _lib
    assert _call("gsr_mip_filter3d", P=-1) == -1
    assert _lib.last_error() == "gsr_mip_filter3d: P and n_cameras must be >= 0"
    assert _call("gsr_mip_filter3d", P=5, n_cameras=-2) == -1
    assert _call("gsr_mip_filter3d", P=0) == 0
    assert _call("gsr_mip_filter3d", P=5, n_cameras=3, cameras=None) == -1
    assert _lib.last_error() == "gsr_mip_filter3d: null pointer"
