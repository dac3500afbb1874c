"""-m gpu: the VisualHull and depth initializers on the device (csrc/gsr_hull.cu, gaustudio_b200.initializers) against
tests/hull_ref64.py: the carved occupancy bit for bit against the float64 restatement and, outside the flagged nodes,
against the reference's own float32 insideView loop run on the same device; the hull mesh's vertices and faces bit for
bit in their documented order; then both initializers end to end."""
import math
import os

import numpy as np
import pytest
import torch

import hull_ref64 as R
import sap_ref64
from gaustudio_b200 import initializers
from gaustudio_b200.camera import look_at_camera
from gaustudio_b200.synthetic import SH_C0, GaussianPointCloud

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
CENTRE, RADIUS = np.array([0.1, -0.2, 0.15]), 0.5


def ring_cameras(n, W, H, dist=4.0, sizes=None):
    """n cameras on two rings (elevations +25 and -35 degrees) looking at the origin; sizes cycles (W, H) pairs."""
    cams = []
    for k in range(n):
        el = math.radians(25.0 if k % 2 == 0 else -35.0)
        az = 2 * math.pi * k / n + 0.3 * (k % 2)
        pos = dist * np.array([math.cos(el) * math.cos(az), math.cos(el) * math.sin(az), math.sin(el)])
        w, h = (W, H) if sizes is None else sizes[k % len(sizes)]
        cams.append(look_at_camera(pos, (0.0, 0.0, 0.0), w, h, 0.9, 0.9 * h / w))
    return cams


def sphere_mask(cam, margin_px=1.5):
    """Pixels whose centre ray passes within the sphere's angular radius plus margin_px pixels: the silhouette, grown
    so that every pixel the sphere's projection touches is set."""
    W, H = cam.image_width, cam.image_height
    K = cam.intrinsics.double().numpy()
    u, v = np.meshgrid(np.arange(W) + 0.5, np.arange(H) + 0.5)
    d = np.stack([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], np.ones_like(u)], -1)
    Rc = np.asarray(cam.R, np.float64)  # camera-to-world rotation
    d = d @ Rc.T
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    c = -Rc @ np.asarray(cam.T, np.float64)
    to = CENTRE - c
    dist = np.linalg.norm(to)
    ang = np.arccos(np.clip(d @ (to / dist), -1, 1))
    return torch.from_numpy(ang <= math.asin(RADIUS / dist) + margin_px / K[0, 0]).to(torch.uint8)


def specs(cams):
    return [(c.full_proj_transform, c.image_width, c.image_height, c.mask) for c in cams]


def check_carve(cams, res, r, t, check32=True):
    occ = initializers.visual_hull_carve(cams, res, r, t)
    x = R.grid_points(res, r, t, DEV)
    dev_specs = [(P.to(DEV), W, H, None if m is None else m.to(DEV)) for P, W, H, m in specs(cams)]
    occ64, flag = R.carve64(x, dev_specs)
    assert torch.equal(occ.reshape(-1).bool(), occ64), "carve differs from the float64 restatement"
    nflag = int(flag.sum())
    if check32:
        occ32 = R.carve32(x, dev_specs)
        bad = (occ32 != occ64) & ~flag
        assert not bool(bad.any()), f"{int(bad.sum())} unflagged nodes differ from the reference's float32 loop"
    return occ, nflag


CASES = {
    "1cam_sphere_128": (1, 128, "sphere", None),
    "7cams_sphere_128": (7, 128, "sphere", None),
    "7cams_nomask_128": (7, 128, None, None),
    "7cams_mixed_sizes_some_unmasked_128": (7, 128, "mixed", [(64, 48), (33, 70), (101, 57)]),
    "300cams_sphere_128": (300, 128, "sphere", None),
    "7cams_sphere_2": (7, 2, "sphere", None),
    "7cams_sphere_512": (7, 512, "sphere", None),
}


@pytest.mark.parametrize("case", list(CASES))
def test_carve_matches_float64_and_the_reference_loop(case):
    n, res, kind, sizes = CASES[case]
    cams = ring_cameras(n, 120, 90, sizes=sizes)
    rng = np.random.default_rng(3)
    for k, c in enumerate(cams):
        if kind == "sphere":
            c.mask = sphere_mask(c)
        elif kind == "mixed" and k % 3 != 2:
            c.mask = torch.from_numpy(rng.uniform(size=(c.image_height, c.image_width)) < 0.97).float()
            c.mask[sphere_mask(c, 0.0).bool()] = 1.0
    r, t = 1.2 * 0.9, np.array([0.03, -0.02, 0.05])
    occ, nflag = check_carve(cams, res, r, t, check32=True)
    assert nflag < 0.02 * res ** 3 + 16
    if kind == "sphere" and res >= 128 and n >= 7:
        x = R.grid_points(res, r, t, DEV).double()
        inside = (x - torch.from_numpy(CENTRE).to(DEV)).norm(dim=1) <= RADIUS
        assert bool(occ.reshape(-1)[inside].bool().all()), "the hull must contain the sphere"
        assert int(occ.sum()) < 3 * int(inside.sum())
    # the same bits again, also after another scene has run
    again = initializers.visual_hull_carve(cams, res, r, t)
    initializers.visual_hull_carve(ring_cameras(3, 50, 40), 64, 2.0, np.zeros(3))
    assert torch.equal(again, occ) and torch.equal(initializers.visual_hull_carve(cams, res, r, t), occ)


def test_carve_with_no_camera_fills_everything():
    occ = initializers.visual_hull_carve([], 16, 1.0, np.zeros(3))
    assert bool((occ == 1).all())


def mesh_case(occ, threshold, r, t):
    v, f = initializers.visual_hull_mesh(occ, threshold, r, t)
    rv, rf, _ = R.hull_mesh64(occ.cpu().numpy(), threshold, r, t)
    assert np.array_equal(v.cpu().numpy(), rv), "vertices differ from the float64 crossing-edge set"
    assert np.array_equal(f.cpu().numpy(), rf), "faces differ"
    return v, f


@pytest.mark.parametrize("threshold", [0.25, 0.5, 0.75])
def test_hull_mesh_vertices_bit_equal_and_closed(threshold):
    cams = ring_cameras(24, 96, 72)
    for c in cams:
        c.mask = sphere_mask(c)
    r, t = 1.1, np.array([0.02, 0.01, -0.03])
    occ = initializers.visual_hull_carve(cams, 64, r, t)
    o = occ.bool()
    assert not (o[0].any() or o[-1].any() or o[:, 0].any() or o[:, -1].any() or o[:, :, 0].any() or
                o[:, :, -1].any()), "the hull must lie strictly inside the grid"
    v, f = mesh_case(occ, threshold, r, t)
    closed, _ = sap_ref64.edge_manifold(f.cpu().numpy())
    assert closed
    assert R.signed_volume(v.cpu().numpy(), f.cpu().numpy()) > 0


@pytest.mark.parametrize("res,p,seed", [(2, 0.5, 0), (3, 0.5, 1), (5, 0.4, 2), (16, 0.5, 3), (33, 0.7, 4)])
def test_hull_mesh_of_random_occupancy(res, p, seed):
    """Every cube case and the grid's border: random occupancies, the mesh bit for bit."""
    g = torch.Generator().manual_seed(seed)
    for k in range(20 if res <= 3 else 2):
        occ = (torch.rand(res, res, res, generator=g) < p).to(torch.uint8).to(DEV)
        if not bool(occ.any()) or bool(occ.all()):
            continue
        mesh_case(occ, (0.25, 0.5, 0.75)[k % 3], 0.8, np.array([0.1, 0.2, -0.3]))


class Dataset(list):
    cameras_center = np.array([0.01, -0.02, 0.0])
    cameras_min_extent = 0.8


def test_visual_hull_initializer_end_to_end(tmp_path, monkeypatch):
    cams = ring_cameras(30, 96, 72)
    for c in cams:
        c.mask = sphere_mask(c)
    init = initializers.make({"name": "VisualHull", "workspace_dir": str(tmp_path), "resolution": 96})
    model = init(GaussianPointCloud.empty(), Dataset(cams))
    r, t = 0.8 * 1.2, Dataset.cameras_center
    occ = initializers.visual_hull_carve(cams, 96, r, t)
    v, f = initializers.visual_hull_mesh(occ, 0.5, r, t)
    assert torch.equal(model._xyz, v)
    P = v.shape[0]
    assert torch.equal(model._opacity, torch.full((P, 1), 0.1, device=DEV))
    assert torch.equal(model._scale, torch.full((P, 3), 0.01, device=DEV))
    assert torch.equal(model._f_dc, torch.zeros(P, 1, 3, device=DEV))
    assert torch.equal(model._rot, torch.tensor([[1.0, 0, 0, 0]], device=DEV).expand(P, 4))
    # the hull contains the sphere: no vertex inside it (beyond one grid step)
    step = 2 * r / 95
    d = (v.double() - torch.from_numpy(CENTRE).to(DEV)).norm(dim=1)
    assert float(d.min()) >= RADIUS - step
    # a second call without overwrite rebuilds the same model from visual_hull.ply
    monkeypatch.setattr(initializers, "visual_hull_carve", lambda *a, **k: pytest.fail("carved again"))
    again = init(GaussianPointCloud.empty(), Dataset(cams))
    for k in ("_xyz", "_opacity", "_scale", "_f_dc", "_rot"):
        assert torch.equal(getattr(again, k), getattr(model, k)), k


def test_visual_hull_from_a_camera_list_uses_getnerfppnorm(tmp_path):
    from gaustudio_b200.extract import getNerfppNorm
    cams = ring_cameras(12, 80, 60)
    for c in cams:
        c.mask = sphere_mask(c)
    model = initializers.make({"name": "VisualHull", "workspace_dir": str(tmp_path), "resolution": 48})(
        GaussianPointCloud.empty(), cams)
    norm = getNerfppNorm(cams)
    occ = initializers.visual_hull_carve(cams, 48, norm["min_radius"] * 1.2, norm["translate"])
    v, _ = initializers.visual_hull_mesh(occ, 0.5, norm["min_radius"] * 1.2, norm["translate"])
    assert torch.equal(model._xyz, v)


def test_empty_hull_raises_before_the_model_is_touched(tmp_path):
    cams = ring_cameras(6, 40, 30)
    for c in cams:
        c.mask = torch.zeros(30, 40)
    model = GaussianPointCloud.empty()
    before = model._xyz
    with pytest.raises(ValueError, match="empty"):
        initializers.make({"name": "VisualHull", "workspace_dir": str(tmp_path), "resolution": 32})(model, cams)
    assert model._xyz is before and not os.path.exists(tmp_path / "visual_hull.ply")


# ---- depth ----
def depth_views(n=5, W=64, H=48):
    """Orbit cameras with the analytic depth of a plane z = -0.6 seen from above-ish, zeros on a stripe, one view
    without depth; images a smooth colour ramp."""
    cams = ring_cameras(n, W, H, dist=3.0)
    for k, c in enumerate(cams):
        if k == 3:
            continue
        K = c.intrinsics.double().numpy()
        u, v = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
        depth = 2.0 + 0.5 * np.sin(u / 9.0 + k) * np.cos(v / 7.0)
        depth[:, 10:13] = 0.0
        c.depth = torch.from_numpy(depth.astype(np.float32))
        img = np.stack([u / W, v / H, 0.5 + 0.5 * np.sin(u * v / 50.0 + k)], -1)
        c.image = torch.from_numpy(np.clip(img, 0, 1).astype(np.float32))
        del K
    return cams


def depth_restatement(cams):
    import copy
    rows = []
    for c in cams:
        if c.depth is None:
            continue
        d = copy.copy(c).downsample_scale(4)
        xyz = d.depth2point(d.depth.to(DEV), coordinate="world").cpu().numpy()
        rows.append((xyz, d.image.numpy(), d.depth.numpy(), d.fx.numpy(), d.fy.numpy()))
    return R.depth_chain(rows)


def test_depth_initializer_matches_the_restatement(tmp_path):
    cams = depth_views()
    before = [(c.image_width, None if c.depth is None else c.depth.clone()) for c in cams]
    init = initializers.make({"name": "depth", "workspace_dir": str(tmp_path)})
    model = init(GaussianPointCloud.empty(), cams)
    for c, (w, d) in zip(cams, before):  # the caller's cameras are untouched
        assert c.image_width == w and (d is None or torch.equal(c.depth, d))
    ref = depth_restatement(cams)
    assert torch.equal(model._xyz.cpu(), torch.from_numpy(ref["xyz"]))
    # colour / 255 on the device, as the reference's build_model divides its CUDA tensor (torch multiplies by the
    # reciprocal there, so this is not the host division of ref["rgb"])
    rgb = torch.from_numpy(ref["colors"]).to(DEV).float() / 255.0
    f_dc = ((rgb - 0.5) / SH_C0).unsqueeze(1)
    assert torch.equal(model._f_dc, f_dc)
    assert torch.equal(model._scale.cpu(), torch.from_numpy(ref["log_scale"]))
    assert bool(torch.isneginf(model._scale).any())  # depth 0: -inf, as in the reference
    assert torch.equal(model._opacity, torch.zeros_like(model._opacity))
    assert model._xyz.shape[0] == 4 * 16 * 12
    # the workspace: fused.ply's colours as written, scales.bin raw float16
    from gaustudio_b200.io import read_ply_vertices
    pv = read_ply_vertices(str(tmp_path / "fused.ply"))
    assert np.array_equal(np.stack([pv[k] for k in ("red", "green", "blue")], 1), ref["colors"])
    assert np.array_equal(np.fromfile(tmp_path / "scales.bin", np.float16), ref["scales16"])
    # rebuilt from the workspace without overwrite
    again = init(GaussianPointCloud.empty(), [])
    for k in ("_xyz", "_f_dc", "_scale", "_opacity"):
        assert torch.equal(getattr(again, k), getattr(model, k)), k
    # without scales.bin the scales come from dist2
    os.remove(tmp_path / "scales.bin")
    d2 = init(GaussianPointCloud.empty(), [])
    want = torch.log(torch.sqrt(initializers.dist2(model._xyz) + 1e-7))[..., None].repeat(1, 3)
    assert torch.equal(d2._scale, want)


def test_depth_initializer_renders_finite(tmp_path):
    from gaustudio_b200 import renderers
    cams = depth_views()
    model = initializers.make({"name": "depth", "workspace_dir": str(tmp_path)})(GaussianPointCloud.empty(), cams)
    r = renderers.make({"name": "vanilla_renderer"})
    for c in ring_cameras(3, 96, 72, dist=3.5):
        with torch.no_grad():
            o = r.render(c.to(DEV), model)
        assert torch.isfinite(o["render"]).all()
        assert float(o["rendered_final_opacity"].max()) > 0
