"""-m gpu: the Mip-Splatting path (2D Mip filter in the projection, 3D smoothing filter, mip_renderer) against the
float64 reference of tests/mip_ref64.py and against the vanilla path.

Bounds as in test_gpu_projection_f64.py: ||a_i - b_i|| <= RTOL ||b_i|| + ATOL max_j ||b_j|| per Gaussian.  Rows whose
float32 decisions are not pinned by the float64 values are left out of the float comparisons: near the lateral clamp
limit, within 1 % of a det0 / det1 clamp, or with an ill-conditioned cov' (a collapsed cov2D at kernel_size 0)."""
import math

import numpy as np
import pytest
import torch

import mip_ref64 as MR
import proj_ref64 as R
from test_gpu_projection_f64 import H, W, dense_sums, isolation_sums, make_scene, precomputed
from test_proj_ref64 import ATOL, NEAR_LIMIT, RTOL

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")


def _collapse(sc, frac, seed):
    """Every 1/frac-th Gaussian gets scales of 1e-7: its cov2D collapses, so det0 (and at k = 0 det1) clamps."""
    sc = dict(sc)
    n = len(sc["means3D"])
    idx = np.arange(0, n, int(round(1 / frac)))
    if "scales" in sc:
        s = sc["scales"].copy()
        s[idx] = 1e-7
        sc["scales"] = s
    else:
        c = sc["cov3D_precomp"].copy()
        c[idx] = np.float32(1e-14) * np.array([1, 0, 0, 1, 0, 1], np.float32)
        sc["cov3D_precomp"] = c
    return sc


def _dev(a):
    return None if a is None else torch.as_tensor(a).to(DEV).contiguous()


def _ref_cam(sc, D, mod):
    c = sc["cam"]
    return R.camera(c.world_view_transform, c.full_proj_transform, c.camera_center, math.tan(c.FoVx * 0.5),
                    math.tan(c.FoVy * 0.5), W, H, D, mod)


def run_mip(sc, D, mod, k, opacities=None, vanilla=False):
    """One forward through the binding: the Mip projection of width k, or (vanilla=True) gsr_forward with `opacities`."""
    from gaustudio_b200 import _C
    c = sc["cam"]
    e = torch.Tensor([])
    T = {key: _dev(sc.get(key)) for key in ("means3D", "shs", "colors_precomp", "opacities", "scales", "rotations",
                                             "cov3D_precomp")}
    if opacities is not None:
        T["opacities"] = opacities.reshape(-1, 1).contiguous()
    g = lambda key: T[key] if T[key] is not None else e
    args = (torch.zeros(3, device=DEV), T["means3D"], g("colors_precomp"), g("opacities"), g("scales"), g("rotations"),
            mod, g("cov3D_precomp"), c.world_view_transform.to(DEV), c.full_proj_transform.to(DEV),
            math.tan(c.FoVx * 0.5), math.tan(c.FoVy * 0.5), H, W, g("shs"), D, c.camera_center.to(DEV), False, False)
    out = _C.rasterize_gaussians(*args) if vanilla else _C.rasterize_gaussians_mip(*args, k)
    R_, color, depth, median, opac, radii, gb, bb, ib = out
    return dict(T=T, radii=radii, gb=gb, bb=bb, ib=ib, R=R_, D=D, mod=mod, k=k, cam=c, images=(color, depth, median, opac))


def _params(fw):
    return {key: v for key, v in fw["T"].items() if v is not None}


def _pinned(f, Dcam):
    """Rows whose float32 decisions follow the float64 values (see the module docstring)."""
    lat = ((f["txtz_over_lim"].abs() - 1).abs() >= NEAR_LIMIT).all(1)
    clamp = ((f["det0"] / MR.EPS6 - 1).abs() > 1e-2) & ((f["det1"] / MR.EPS6 - 1).abs() > 1e-2)
    a, b, c = f["cov2D"].unbind(1)
    cond = (a * c - b * b) > 1e-3 * a * c
    return (lat & clamp & cond).numpy()


def _near_int(x, tol=1e-4):
    x = np.asarray(x, np.float64)
    return np.abs(x - np.round(x)) <= tol


FWD_CASES = [pytest.param(k, D, pre, mod, id=f"k{k}-D{D}-{'precomp' if pre else 'sh'}-mod{mod}")
             for k in (0.0, 0.1, 0.3, 2.0) for D, pre, mod in ((0, False, 1.0), (1, False, 1.3), (3, False, 1.0),
                                                               (0, True, 1.3))]


@pytest.mark.parametrize("k,D,pre,mod", FWD_CASES)
def test_forward_records_against_f64_reference(k, D, pre, mod):
    """means2D, conic, o', depth and rgb of every splat, radii and tiles touched, read back with gsr_debug_export."""
    from gaustudio_b200 import _C
    P = 3001
    sc = make_scene(P, 16, 300 + D + int(10 * k), False)
    if pre:
        sc = precomputed(sc)
    sc = _collapse(sc, 0.05, 7)
    fw = run_mip(sc, D, mod, k)
    Dcam = _ref_cam(sc, D, mod)
    f = MR.forward(_params(fw), Dcam, k)
    ex = _C.debug_export(P, W, H, fw["R"], fw["gb"], fw["bb"], fw["ib"])
    radii = fw["radii"].cpu().numpy()
    pinned = _pinned(f, Dcam)
    near_ceil = _near_int(f["pre_ceil"].numpy())
    # integer outputs: exact, except where the float64 value under the ceil is within 1e-4 of a jump
    sure = pinned & ~near_ceil
    assert np.array_equal(radii[sure], f["radius"].numpy()[sure]), "radii"
    vis = radii > 0
    px = f["means2D"][:, 0].numpy()
    py = f["means2D"][:, 1].numpy()
    rr = radii.astype(np.float64)
    edges = [(px - rr) / 16, (px + rr + 15) / 16, (py - rr) / 16, (py + rr + 15) / 16]
    rect_sure = sure & vis & ~np.any([_near_int(e) for e in edges], axis=0)
    ref_tiles = ((f["rect"][:, 2] - f["rect"][:, 0]) * (f["rect"][:, 3] - f["rect"][:, 1])).numpy()
    tt = ex["tiles_touched"].cpu().numpy()
    assert np.array_equal(tt[rect_sure], ref_tiles[rect_sure]), "tiles touched"
    m = vis & pinned
    assert m.sum() > 1000, m.sum()
    co = ex["conic_opacity"].cpu()
    pairs = (("means2D", ex["means2D"].cpu(), f["means2D"]), ("conic", co[:, :3], f["conic"]),
             ("opacity", co[:, 3:4], f["opacity"][:, None]), ("depth", ex["depths"].cpu(), f["depth"]),
             ("rgb", ex["rgb"].cpu(), f["rgb"] if not pre else R.t64(sc["colors_precomp"])))
    for name, a, b in pairs:
        r, i, n = R.row_check(a, b, RTOL, ATOL, m)
        assert r <= 1, f"k={k} D={D}: {name} row {i} at {r:.3g} x the bound ({n} rows over)"
    # collapsed Gaussians: the det0 clamp fired, so they carry opacity exactly 0 (and bin no tile)
    col = vis & (f["det0"].numpy() < 0.5e-6)
    assert col.sum() > 20, col.sum()
    assert (co[:, 3].numpy()[col] == 0).all()
    if k == 0.0:  # cov' = cov2D: a collapsed Gaussian's det is 0 or tiny, and only the clamp keeps it invisible
        assert (f["det1"].numpy()[col] < 0.5e-6).all()


@pytest.mark.parametrize("pre", [False, True], ids=["sh", "precomp"])
def test_k03_matches_the_vanilla_forward_given_the_filtered_opacities(pre):
    """At kernel_size 0.3, cov' is the vanilla path's dilated cov2D, so gsr_forward fed the splats' o' must give the
    same radii, rects, binned list and images."""
    from gaustudio_b200 import _C
    P = 20000
    sc = make_scene(P, 16, 41, False)
    if pre:
        sc = precomputed(sc)
    sc = _collapse(sc, 0.02, 3)
    a = run_mip(sc, 3, 1.0, 0.3)
    ea = _C.debug_export(P, W, H, a["R"], a["gb"], a["bb"], a["ib"])
    b = run_mip(sc, 3, 1.0, None, opacities=ea["conic_opacity"][:, 3].clone(), vanilla=True)
    eb = _C.debug_export(P, W, H, b["R"], b["gb"], b["bb"], b["ib"])
    assert torch.equal(a["radii"], b["radii"]) and a["R"] == b["R"]
    for key in ("tiles_touched", "ranges", "point_list", "n_contrib", "means2D", "conic_opacity", "depths", "rgb"):
        assert torch.equal(ea[key], eb[key]), key
    for x, y in zip(a["images"], b["images"]):
        assert float((x - y).abs().max()) <= 1e-6
        assert torch.equal(x, y)  # the geometry code is shared: bit-identical


BWD_CASES = [pytest.param(k, pre, P, id=f"k{k}-{'precomp' if pre else 'sh16'}-P{P}")
             for k, pre, P in ((0.1, False, 1061), (0.3, False, 20000), (2.0, False, 128), (0.3, True, 1061),
                               (0.0, False, 1061))]


@pytest.mark.parametrize("k,pre,P", BWD_CASES)
def test_projection_backward_against_f64_vjp(k, pre, P):
    """The Mip projection backward alone (gsr_debug_projection_backward_mip) on dense and isolated sums, every output
    against the float64 VJP; culled Gaussians and Gaussians without sums get exact zeros."""
    from gaustudio_b200 import _C
    D, mod = (0, 1.3) if pre else (3, 1.0)
    seed = 900 + P + int(10 * k)
    sc = make_scene(P, 16, seed, False)
    if pre:
        sc = precomputed(sc)
    sc = _collapse(sc, 0.02, 5)
    fw = run_mip(sc, D, mod, k)
    Dcam = _ref_cam(sc, D, mod)
    params = _params(fw)
    radii = fw["radii"].cpu().numpy()
    vis = radii > 0
    ex = _C.debug_export(P, W, H, fw["R"], fw["gb"], fw["bb"], fw["ib"])
    clamped = ex["clamped"].cpu().numpy().astype(bool)
    f = MR.forward(params, Dcam, k)
    pinned = _pinned(f, Dcam)
    T, c = fw["T"], fw["cam"]
    keys = dict(mean2D="mean2D", conic="conic", opacity="opacity", color="color", depth="depth", mean3D="means3D",
                cov3D="cov3D")
    if not pre:
        keys.update(shs="shs", scale="scales", rot="rotations")
    for kind, sums in (("dense", dense_sums(P, seed)), ("isolated", isolation_sums(P, seed))):
        for pname, pat in (("all", np.ones(P, bool)), ("every3", np.arange(P) % 3 == 1)):
            s = torch.where(torch.as_tensor(pat)[:, None], sums, torch.zeros_like(sums))
            up = MR.upstream_from_sums(s, params, Dcam, k, radii)
            ref = MR.vjp(params, Dcam, k, up, radii, clamped)
            out = _C.debug_projection_backward_mip(
                T["means3D"], T["shs"], T["colors_precomp"], T["opacities"], T["scales"], mod, T["rotations"],
                T["cov3D_precomp"], c.world_view_transform.to(DEV), c.full_proj_transform.to(DEV),
                c.camera_center.to(DEV), math.tan(c.FoVx * 0.5), math.tan(c.FoVy * 0.5), H, W, D, fw["radii"],
                fw["gb"], s, k)
            torch.cuda.synchronize()
            live = pat & vis & (s[:, :10] != 0).any(1).numpy()
            what = f"k={k} P={P} {kind}/{pname}"
            for ok, a in out.items():
                a = a.cpu()
                assert torch.isfinite(a).all(), f"{what}: {ok} not finite"
                assert not a[torch.as_tensor(~live)].any(), f"{what}: {ok} non-zero without a gradient"
                if ok not in keys:
                    assert not a.any(), f"{what}: {ok} should be zero"
                    continue
                r, i, n = R.row_check(a, ref[keys[ok]], RTOL, ATOL, live & pinned)
                assert r <= 1, f"{what}: {ok} row {i} at {r:.3g} x the bound ({n} rows over)"


def _filter_scene(P, C, seed):
    from gaustudio_b200.camera import look_at_camera
    rng = np.random.RandomState(seed)
    xyz = rng.randn(P, 3) * 1.5
    xyz[:50] = rng.randn(50, 3) * 200.0       # far away: many views miss them
    xyz[50:60] = rng.randn(10, 3) * 1e-3
    xyz[60:70] = np.stack([3e5 + 1e4 * rng.rand(10), 1e3 * rng.randn(10), 1e3 * rng.randn(10)], 1)  # d capped at 1e5
    xyz[70:90] = np.stack([rng.randn(20), rng.randn(20), 1e4 + rng.rand(20)], 1)  # above and behind every camera
    cams = []
    for i in range(C):
        d = rng.randn(3)
        d[2] = abs(d[2]) + 0.3  # the upper half: every camera looks down at the origin
        d /= np.linalg.norm(d)
        pos = d * (3.0 + 6.0 * rng.rand())
        tgt = rng.randn(3) * 0.5
        Wc, Hc = int(rng.choice([64, 320, 1920])), int(rng.choice([48, 240, 1080]))
        fov = math.radians(30 + 50 * rng.rand())
        cams.append(look_at_camera(pos, tgt, Wc, Hc, fov, fov * Hc / Wc))
    # one camera looking along +x, at the Gaussians ~3e5 away: their d is capped at 100000
    cams.append(look_at_camera((-10.0, 0.0, 0.0), (0.0, 0.0, 0.0), 640, 480, 0.5, 0.4))
    return xyz.astype(np.float32), cams


def _filter_count(xyz, recs):
    from gaustudio_b200 import _lib
    out = torch.empty(xyz.shape[0], device=DEV)
    scratch = torch.empty(3, dtype=torch.int32, device=DEV)
    rc = _lib.lib().gsr_mip_filter3d(xyz.shape[0], xyz.data_ptr(), recs.shape[0], recs.data_ptr(), out.data_ptr(),
                                     scratch.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _lib.last_error()
    return out, int(scratch[2])


def test_filter3d_against_f64_oracle():
    """1,001 cameras (four shared-memory chunks) and P not a multiple of the block size."""
    from gaustudio_b200 import _C
    P = 20011
    xyz, cams = _filter_scene(P, 1000, 5)
    # the oracle reads the float32 records the kernel gets (R and T rounded), in float64
    recs64 = _C.mip_camera_records(cams, torch.device("cpu")).double().numpy()
    assert np.abs(recs64 - MR.camera_records(cams)).max() <= 1e-6 * np.abs(MR.camera_records(cams)).max()
    ref, seen = MR.filter3d(xyz, recs64)
    near = MR.near_boundary(xyz, recs64)
    x = torch.from_numpy(xyz).to(DEV)
    got = _C.mip_filter3d(x, cams).cpu().numpy().astype(np.float64)
    again = _C.mip_filter3d(x, cams).cpu().numpy().astype(np.float64)
    assert np.array_equal(got, again), "two runs differ"
    ok = ~near
    assert ok.sum() > 0.9 * P and (~seen[ok]).sum() > 10 and seen[ok].sum() > 1000
    rel = np.abs(got - ref) / np.abs(ref)
    assert rel[ok].max() <= 1e-6, (rel[ok].max(), int(np.argmax(np.where(ok, rel, 0))))
    capped = seen & (ref >= 100000.0 / recs64[:, 12].max() * math.sqrt(0.2) * (1 - 1e-12))
    assert capped[ok].sum() >= 1
    # the seen count: exact up to the Gaussians at a visibility boundary
    recs = _C.mip_camera_records(cams, DEV)
    _, n = _filter_count(x, recs)
    assert abs(n - int(seen.sum())) <= int(near.sum())


def test_filter3d_raises_when_nothing_is_seen():
    from gaustudio_b200 import _C
    from gaustudio_b200.camera import look_at_camera
    cams = [look_at_camera((5.0, 0.0, 0.0), (0.0, 0.0, 0.0), 64, 48, 0.6, 0.45)]
    x = torch.tensor([[10.0, 0.0, 0.0], [6.0, 0.0, 0.0], [0.0, 50.0, 0.0]], device=DEV)  # behind, too near, off-screen
    with pytest.raises(ValueError, match="no camera sees"):
        _C.mip_filter3d(x, cams)
    from gaustudio_b200.mip import MipPointCloud
    m = MipPointCloud(x, torch.zeros(3, 3, device=DEV), torch.tensor([[1.0, 0, 0, 0]] * 3, device=DEV),
                      torch.zeros(3, 1, device=DEV), torch.zeros(3, 1, 3, device=DEV), torch.zeros(3, 15, 3, device=DEV))
    with pytest.raises(ValueError):
        m.compute_3D_filter(cams)


# ---- buffers that hold another scene's state ------------------------------------------------------------------------
class _Bufs:
    """Allocator callback that hands out caller-seeded buffers (one per slot), grown only when too small."""

    def __init__(self, seeds=None):
        from gaustudio_b200 import _lib
        self.seeds = seeds or {}
        self.bufs = {}
        self.fn = _lib.ALLOC_FN(self._alloc)

    def _alloc(self, user, n):
        seed = self.seeds.get(user)
        t = torch.zeros(int(n), dtype=torch.uint8, device=DEV)
        if seed is not None:
            m = min(seed.numel(), t.numel())
            t[:m] = seed[:m]
        self.bufs[user] = t
        return t.data_ptr()


def _fwd_bwd(fw_in, k, bufs, fill):
    from gaustudio_b200 import _C, _lib
    L = _lib.lib()
    T, c, D = fw_in["T"], fw_in["cam"], fw_in["D"]
    P = T["means3D"].shape[0]
    p = _C._ptr
    outs = [torch.full(s, fill, device=DEV) for s in ((3, H, W), (1, H, W), (3, H, W), (1, H, W))]
    radii = torch.full((P,), -7, dtype=torch.int32, device=DEV)
    view, proj, campos = (x.to(DEV).contiguous() for x in (c.world_view_transform, c.full_proj_transform,
                                                          c.camera_center))
    bg = torch.zeros(3, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    Rn = L.gsr_forward_mip(bufs.fn, 1, bufs.fn, 2, bufs.fn, 3, P, D, 16, p(bg), W, H, p(T["means3D"]), p(T["shs"]), None,
                           p(T["opacities"]), p(T["scales"]), 1.0, p(T["rotations"]), None, p(view), p(proj), p(campos),
                           math.tan(c.FoVx * 0.5), math.tan(c.FoVy * 0.5), 0, *[p(o) for o in outs], p(radii), 0, 0, None,
                           float(k), st)
    assert Rn >= 0, _lib.last_error()
    g = torch.Generator().manual_seed(3)
    dpix = [torch.randn(o.shape, generator=g).to(DEV) for o in outs]
    grads = dict(m2=(P, 3), conic=(P, 4), op=(P,), col=(P, 3), depth=(P,), m3=(P, 3), cov=(P, 6), sh=(P, 16, 3),
                 sc=(P, 3), rot=(P, 4))
    gr = {key: torch.full(s, fill, device=DEV) for key, s in grads.items()}
    rc = L.gsr_backward_mip(P, D, 16, Rn, p(bg), W, H, p(T["means3D"]), p(T["shs"]), None, p(T["scales"]), 1.0,
                            p(T["rotations"]), None, p(view), p(proj), p(campos), math.tan(c.FoVx * 0.5),
                            math.tan(c.FoVy * 0.5), p(radii), p(bufs.bufs[1]), p(bufs.bufs[2]), p(bufs.bufs[3]),
                            *[p(d) for d in dpix], p(gr["m2"]), p(gr["conic"]), p(gr["op"]), p(gr["col"]),
                            p(gr["depth"]), p(gr["m3"]), p(gr["cov"]), p(gr["sh"]), p(gr["sc"]), p(gr["rot"]), 0,
                            p(T["opacities"]), float(k), st)
    assert rc == 0, _lib.last_error()
    torch.cuda.synchronize()
    from gaustudio_b200 import _C as C_
    ex = C_.debug_export(P, W, H, Rn, bufs.bufs[1], bufs.bufs[2], bufs.bufs[3])
    return Rn, outs, radii, ex, gr


def test_no_dependence_on_earlier_buffer_contents():
    """A Mip forward and backward on buffers that hold a full forward + backward of another scene (same P, W, H), with
    NaN-filled outputs, gives bitwise the fresh forward and the fresh gradients up to float-atomic summation order."""
    from gaustudio_b200 import _C
    P, k = 6000, 0.3
    prev = _C.set_speculation(False)  # one binning allocation per forward: the seeded one
    try:
        donor = run_mip(make_scene(P, 16, 11, False), 3, 1.0, k)
        d_bufs = _Bufs()
        _fwd_bwd(donor, k, d_bufs, 0.0)
        seeds = {u: t.clone() for u, t in d_bufs.bufs.items()}
        target = run_mip(make_scene(P, 16, 12, False), 3, 1.0, k)
        fresh = _fwd_bwd(target, k, _Bufs(), 0.0)
        stale = _fwd_bwd(target, k, _Bufs(seeds), float("nan"))
    finally:
        _C.set_speculation(prev)
    assert fresh[0] == stale[0]
    for x, y in zip(fresh[1], stale[1]):
        assert torch.equal(x, y)
    assert torch.equal(fresh[2], stale[2])
    for key in ("point_list", "ranges", "n_contrib", "final_T", "means2D", "conic_opacity", "depths", "rgb"):
        assert torch.equal(fresh[3][key], stale[3][key]), key
    for key in fresh[4]:
        x, y = fresh[4][key], stale[4][key]
        assert torch.isfinite(y).all(), key
        assert float((x - y).abs().max()) <= 1e-5 * float(x.abs().max()) + 1e-12, key


# ---- end to end -----------------------------------------------------------------------------------------------------
def _mip_model(n=4000, seed=0, radius=0.5, device="cuda"):
    from gaustudio_b200.mip import MipPointCloud
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(n, 3, generator=g)
    xyz = radius * d / d.norm(dim=1, keepdim=True)
    scale = math.log(0.02) + 0.2 * torch.randn(n, 3, generator=g)
    rot = torch.randn(n, 4, generator=g)
    opacity = 2.0 + 0.5 * torch.randn(n, 1, generator=g)
    f_dc = torch.randn(n, 1, 3, generator=g)
    f_rest = 0.1 * torch.randn(n, 15, 3, generator=g)
    return MipPointCloud(xyz, scale, rot, opacity, f_dc, f_rest, 3, 3).to(device)


def _cams(n=12, W=128, H=96):
    from gaustudio_b200.camera import orbit_cameras
    fov = math.radians(50.0)
    return (orbit_cameras(n, 2.0, 20.0, W, H, 2 * math.atan(math.tan(fov / 2) * W / H), fov) +
            orbit_cameras(n // 2, 2.0, -40.0, W, H, 2 * math.atan(math.tan(fov / 2) * W / H), fov))


def test_mip_renderer_renders_an_exported_mip_ply(tmp_path):
    from gaustudio_b200 import io, renderers
    from gaustudio_b200.mip import MipPointCloud
    model = _mip_model()
    cams = _cams()
    model.compute_3D_filter(cams)
    assert model.filter_3D.shape == (model.num_points, 1) and bool((model.filter_3D > 0).all())
    path = str(tmp_path / "mip.ply")
    io.export_ply(model, path)
    loaded = io.load_ply(path, active_sh_degree=3, device="cuda")
    assert isinstance(loaded, MipPointCloud)
    assert torch.equal(loaded.filter_3D, model.filter_3D)
    cam = cams[0].to("cuda")
    base = renderers.make({"name": "mip_renderer"}).render(cam, loaded)
    assert set(base) == {"render", "rendered_depth", "rendered_median_depth", "rendered_median_weight",
                         "rendered_median_id", "viewspace_points", "visibility_filter", "rendered_final_opacity",
                         "radii"}
    assert float(base["rendered_final_opacity"].max()) > 0.9
    for opt in ("compute_cov3D_python", "convert_SHs_python"):
        other = renderers.make({"name": "mip_renderer", opt: True}).render(cam, loaded)
        diff = float((other["render"] - base["render"]).abs().max())
        assert diff <= 1e-5, (opt, diff)
    # kernel_size changes the picture: the Mip filter is really in the path
    wide = renderers.make({"name": "mip_renderer", "kernel_size": 2.0}).render(cam, loaded)
    assert float((wide["render"] - base["render"]).abs().max()) > 1e-3
    # a model without filter_3D is refused before any device work
    plain = MipPointCloud.from_model(loaded)
    with pytest.raises(ValueError, match="compute_3D_filter"):
        renderers.make("mip_renderer").render(cam, plain)


def test_training_with_the_mip_renderer_lowers_the_loss():
    """200 Adam steps fit perturbed parameters to a target rendered from the true ones: the loss drops 4x."""
    from gaustudio_b200 import optimizers, renderers
    r = renderers.make({"name": "mip_renderer", "kernel_size": 0.1})
    cams = [c.to("cuda") for c in _cams(8, 96, 72)]
    target_model = _mip_model(n=1500, seed=4)
    target_model.compute_3D_filter(cams)
    with torch.no_grad():
        targets = [r.render(c, target_model)["render"] for c in cams]
    model = _mip_model(n=1500, seed=4)
    g = torch.Generator(device="cuda").manual_seed(9)
    model._f_dc = model._f_dc + 0.5 * torch.randn(model._f_dc.shape, generator=g, device="cuda")
    model._opacity = model._opacity - 1.5
    model._scale = model._scale + 0.3 * torch.randn(model._scale.shape, generator=g, device="cuda")
    model.compute_3D_filter(cams)
    model.requires_grad_(True)
    opt = optimizers.make({"name": "general", "model": model, "optimizer_name": "Adam", "args": {"lr": 0.0, "eps": 1e-15},
                           "params": {"opacity": {"lr": 0.05}, "f_dc": {"lr": 0.01}, "scale": {"lr": 0.005}}})
    losses = []
    for it in range(200):
        c, t = cams[it % len(cams)], targets[it % len(cams)]
        loss = (r.render(c, model)["render"] - t).abs().mean()
        loss.backward()
        opt.step()
        opt.zero_grad()
        losses.append(float(loss))
    first, last = np.mean(losses[:8]), np.mean(losses[-8:])
    print(f"\nmip fit: L1 {first:.4g} -> {last:.4g} ({first / last:.1f}x)")
    assert last < first / 4, (first, last)


def test_extract_mesh_with_the_mip_renderer():
    from gaustudio_b200 import mesh, renderers
    r = renderers.make("mip_renderer")
    model = _mip_model(n=8000, seed=2)
    cams = _cams(16, 128, 96)
    model.compute_3D_filter(cams)
    vs = 0.02
    V, F = mesh.extract_mesh(r, model, cams, voxel_size=vs, sdf_trunc=3 * vs, min_weight=1)
    assert F.shape[0] > 1000, F.shape
    rad = V.norm(dim=1)
    assert float((rad - 0.5).abs().median()) < 1.5 * vs, float((rad - 0.5).abs().median())
