"""Surfel rasterizer on the GPU (csrc/gsr_surfel.cu) against the float64 contract of tests/surfel_ref64.py, plus
determinism, independence from stale buffer contents, the extraction flows end to end and a short training run."""
import math

import numpy as np
import pytest
import torch

import surfel_ref64 as ref
import surfel_scenes as ss
from gaustudio_b200 import _C, _lib

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _inputs(s, grads=False):
    f = lambda k: torch.tensor(s[k], device=DEV)
    t = {k: f(k).requires_grad_(grads) for k in ("means3D", "scales", "rotations", "opacities", "shs", "colors_precomp")
         if k in s}
    return t


def _settings(s, debug=False):
    from gaustudio_b200.surfel_rasterizer import GaussianRasterizationSettings
    f = lambda k: torch.tensor(s[k], device=DEV)
    return GaussianRasterizationSettings(s["H"], s["W"], s["tanfovx"], s["tanfovy"], f("bg"), s["scale_modifier"],
                                         f("viewmatrix"), f("projmatrix"), s["D"], f("campos"), False, debug)


def gpu_run(s, upstream=None):
    """-> (color[3,H,W], radii, allmap[9,H,W], grads dict or None)."""
    from gaustudio_b200.surfel_rasterizer import GaussianRasterizer
    t = _inputs(s, upstream is not None)
    m2 = torch.zeros_like(t["means3D"], requires_grad=upstream is not None)
    color, radii, allmap = GaussianRasterizer(_settings(s))(
        t["means3D"], m2, t["opacities"], shs=t.get("shs"), colors_precomp=t.get("colors_precomp"),
        scales=t["scales"], rotations=t["rotations"])
    grads = None
    if upstream is not None:
        gi, gm = upstream
        ((color * gi).sum() + (allmap * gm).sum()).backward()
        grads = {k: v.grad for k, v in t.items()}
        grads["means2D"] = m2.grad
    return color.detach(), radii, allmap.detach(), grads


def raw_forward(s):
    """_C.rasterize_surfels -> (R, color, radii, allmap, geom, binning, image)."""
    f = lambda k: torch.tensor(s[k], device=DEV)
    e = torch.empty(0, device=DEV)
    return _C.rasterize_surfels(f("bg"), f("means3D"), f("colors_precomp") if "colors_precomp" in s else e,
                                f("opacities"), f("scales"), f("rotations"), s["scale_modifier"], f("viewmatrix"),
                                f("projmatrix"), s["tanfovx"], s["tanfovy"], s["H"], s["W"],
                                f("shs") if "shs" in s else e, s["D"], f("campos"), False, False)


def _geom_records(geom, P):
    """mean2D [P,2] and packed tile rects [P,4] from the surfel geometry buffer (layout of csrc/gsr_surfel.cu)."""
    from test_gpu_surfel_f64 import geom_views
    v = geom_views(geom, P)
    recA, rect = v["recA"], v["rect"]
    r = torch.stack([rect[:, 0] & 0xffff, rect[:, 1] & 0xffff, (rect[:, 0] >> 16) & 0xffff, (rect[:, 1] >> 16) & 0xffff], 1)
    return recA[:, 0:2], r


def _pix_of(o, H, W):
    return o["pix"][:, 1].cpu() * W + o["pix"][:, 0].cpu()


def check_forward(s, pix=None, what=""):
    R, color, radii, allmap, geom, _, _ = raw_forward(s)
    o = ref.run(s, device=DEV, pix=pix)
    g = o["geom"]
    H, W, P = s["H"], s["W"], s["means3D"].shape[0]
    # radii and rects exact (Gaussians whose radius sits within rounding of an integer excepted)
    rc, live = ref.rects(g)
    exact = ~g["rad_amb"]
    assert torch.equal(radii.long()[exact], torch.where(live, g["radius"], torch.zeros_like(g["radius"])).long()[exact]), what
    m2, grect = _geom_records(geom, P)
    lv = (radii > 0) & exact
    near_edge = torch.zeros_like(lv)
    for c in range(2):  # a centre within 1e-3 px of making (c -/+ r)/16 an integer is allowed to land either side
        for sgn, add in ((-1, 0), (1, 15)):
            v = (g["mx" if c == 0 else "my"].detach() + sgn * g["radius"] + add) / 16
            near_edge |= ((v - torch.round(v)).abs() < 1e-3 / 16)
    sel = lv & ~near_edge
    assert torch.equal(grect.long()[sel], rc[sel]), what
    assert int(R) == int(((rc[:, 2] - rc[:, 0]) * (rc[:, 3] - rc[:, 1]))[live].sum()) or bool(near_edge[live].any())
    torch.testing.assert_close(m2[sel].double(), torch.stack([g["mx"], g["my"]], 1)[sel].detach(), rtol=1e-4, atol=2e-3)
    # images on unflagged pixels
    idx = _pix_of(o, H, W).to(DEV)
    ok = ~o["flag"]
    # grazing splats flag a wide band where rho3 ~ rho2 (near-parallel rays make s imprecise): most pixels still count
    # (small images: one ambiguous rect edge flags a whole tile band)
    assert ok.float().mean() > 0.3 and int((ok & (o["maps"][1] > 0.05)).sum()) >= 15, (what, float(ok.float().mean()))
    gi = color.reshape(3, -1)[:, idx].double()
    gm = allmap.reshape(9, -1)[:, idx].double()
    err = lambda a, b: float((a[:, ok] - b[:, ok]).abs().max()) if ok.any() else 0.0
    assert err(gi, o["image"]) < 1e-4, (what, "image", err(gi, o["image"]))
    for c, name in ((0, "depth"), (1, "alpha"), (2, "normal"), (3, "normal"), (4, "normal"), (5, "median depth")):
        e = err(gm[c:c + 1], o["maps"][c:c + 1])
        # expected depth D = sum w z: z up to ~4 here, so its bound scales with the depth
        bound = 1e-4 * max(1.0, float(o["maps"][5].abs().max())) if c == 0 else 1e-4
        assert e < bound, (what, name, e)
    assert torch.equal(gm[8][ok], o["maps"][8][ok]), what  # median id exact
    assert torch.equal(gm[7][ok] == 0, o["maps"][7][ok] == 0), what
    dref = o["maps"][6][ok]
    assert float((gm[6][ok] - dref).abs().max()) <= 1e-3 * float(dref.abs().max()) + 1e-6, what  # distortion
    return o


CASES = [(n, dict(D=d)) for n in ss.SCENES for d in (0, 3)] + [
    ("random", dict(D=1)), ("random", dict(D=2)), ("sphere", dict(colors=True)), ("stacks", dict(colors=True)),
    ("random", dict(bg=(1.0, 1.0, 1.0))), ("grazing", dict(bg=(1.0, 1.0, 1.0), colors=True)),
    ("random", dict(scale_modifier=0.7)), ("sphere", dict(scale_modifier=1.4, W=97, H=33)),
    ("stacks", dict(W=16, H=16)), ("random", dict(W=33, H=17)), ("near", dict(W=100, H=75))]


@pytest.mark.parametrize("name,kw", CASES, ids=[f"{n}-{'-'.join(f'{k}{v}' for k, v in kw.items())}" for n, kw in CASES])
def test_forward_matches_float64_contract(name, kw):
    check_forward(ss.scene(name, **kw), what=name)


def test_forward_1080p_sampled_tiles():
    s = ss.scene("random", W=1920, H=1080, P=100000, s0=0.01)
    R, color, radii, allmap, *_ = raw_forward(s)
    assert int((radii > 0).sum()) > 90000
    gx = (1920 + 15) // 16
    alpha_t = torch.nn.functional.avg_pool2d(allmap[1:2, :1072], 16).flatten()
    busy = torch.argsort(alpha_t, descending=True)[:4].tolist()
    rng = np.random.RandomState(3)
    tiles = busy + [int(t) for t in rng.choice(int((alpha_t > 0.05).sum()), 2)] + [gx * 67 + 119]  # + the last tile
    pix = []
    for t in tiles:
        ty, tx = divmod(t, gx)
        for y in range(ty * 16, min(ty * 16 + 16, 1080)):
            for x in range(tx * 16, min(tx * 16 + 16, 1920)):
                pix.append((x, y))
    check_forward(s, pix=torch.tensor(pix, device=DEV), what="1080p")


def _upstream(s, n_pix, seed=7):
    g = torch.Generator().manual_seed(seed)
    gi = torch.randn(3, n_pix, generator=g, dtype=torch.float64)
    gm = torch.randn(7, n_pix, generator=g, dtype=torch.float64)
    return gi.to(DEV), gm.to(DEV)


BWD = [("random", {}), ("sphere", {}), ("grazing", {}), ("near", {}), ("stacks", {}), ("random", dict(colors=True)),
       ("stacks", dict(D=1, bg=(1.0, 1.0, 1.0))), ("random", dict(scale_modifier=0.8, W=40, H=37))]


@pytest.mark.parametrize("name,kw", BWD, ids=[f"{n}-{'-'.join(f'{k}{v}' for k, v in kw.items())}" for n, kw in BWD])
def test_backward_matches_float64_autograd(name, kw):
    s = ss.scene(name, **kw)
    H, W = s["H"], s["W"]
    gi, gm = _upstream(s, H * W)
    o = ref.run(s, device=DEV, grads=True, upstream=(gi, gm))
    keep = (~o["flag"]).double()
    up = ((gi * keep).float().reshape(3, H, W), torch.cat([(gm * keep).float(), torch.zeros(2, H * W, device=DEV)]).reshape(9, H, W))
    _, radii, _, grads = gpu_run(s, upstream=up)
    pairs = [("means3D", "means3D"), ("scales", "scales"), ("rotations", "rotations"), ("opacities", "opacities"),
             ("shs" if "shs" in s else "colors_precomp",) * 2]
    for gk, rk in pairs:
        a, b = grads[gk].double(), o["grads"][rk]
        scale = float(b.abs().max())
        assert scale > 0, gk
        assert float((a - b).abs().max()) <= 1e-3 * scale, (name, gk, float((a - b).abs().max()), scale)
    a, b = grads["means2D"][:, :2].double(), o["grads"]["means2D"]
    assert float((a - b).abs().max()) <= 1e-3 * float(b.abs().max()), (name, "means2D")
    assert float(grads["means2D"][:, 2].abs().max()) == 0.0
    dead = radii == 0  # culled Gaussians get exact zeros
    for v in grads.values():
        assert float(v[dead].abs().max()) == 0.0 if bool(dead.any()) else True


# ---- determinism and stale buffers ------------------------------------------------------------------------------------
def _forward_with(s, fill):
    """gsr_surfel_forward through the C ABI with buffers pre-filled by `fill(slot, nbytes)`; outputs pre-filled with NaN."""
    L = _lib.lib()
    bufs = {}

    def alloc(user, n):
        bufs[user] = fill(user, int(n))
        return bufs[user].data_ptr()

    A = _lib.ALLOC_FN(alloc)
    t = _inputs(s)
    cam = {k: torch.tensor(s[k], device=DEV) for k in ("bg", "viewmatrix", "projmatrix", "campos")}  # alive for the call
    f = lambda k: cam[k]
    P, H, W = s["means3D"].shape[0], s["H"], s["W"]
    color = torch.full((3, H, W), float("nan"), device=DEV)
    amap = torch.full((9, H, W), float("nan"), device=DEV)
    radii = torch.full((P,), -7, dtype=torch.int32, device=DEV)
    sh = t.get("shs")
    r = L.gsr_surfel_forward(A, 1, A, 2, A, 3, P, s["D"], sh.shape[1] if sh is not None else 0, f("bg").data_ptr(), W, H,
                             t["means3D"].data_ptr(), sh.data_ptr() if sh is not None else None,
                             t["colors_precomp"].data_ptr() if "colors_precomp" in t else None,
                             t["opacities"].data_ptr(), t["scales"].data_ptr(), s["scale_modifier"],
                             t["rotations"].data_ptr(), f("viewmatrix").data_ptr(), f("projmatrix").data_ptr(),
                             f("campos").data_ptr(), 0, color.data_ptr(), amap.data_ptr(), radii.data_ptr(), 0,
                             torch.cuda.current_stream().cuda_stream)
    assert r >= 0, _lib.last_error()
    torch.cuda.synchronize()
    return r, color, amap, radii, bufs


@pytest.mark.parametrize("name", ["random", "stacks"])
def test_forward_is_deterministic_and_ignores_stale_buffers(name):
    s = ss.scene(name, W=70, H=50)
    donor = ss.scene(name, W=70, H=50, seed=99)
    *_, dbufs = _forward_with(donor, lambda u, n: torch.zeros(n, dtype=torch.uint8, device=DEV))
    runs = {
        "zero": lambda u, n: torch.zeros(n, dtype=torch.uint8, device=DEV),
        "nan": lambda u, n: torch.full((n,), 0xFF, dtype=torch.uint8, device=DEV),
        "foreign": lambda u, n: dbufs[u][:n].clone() if dbufs[u].numel() >= n else
        torch.cat([dbufs[u], torch.full((n - dbufs[u].numel(),), 0x7F, dtype=torch.uint8, device=DEV)]),
    }
    base = _forward_with(s, runs["zero"])
    again = _forward_with(s, runs["zero"])
    for k in runs:
        other = _forward_with(s, runs[k]) if k != "zero" else again
        assert other[0] == base[0], k
        for a, b in zip(base[1:4], other[1:4]):
            assert torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a,
                               b.view(torch.int32) if b.dtype == torch.float32 else b), k
    assert not torch.isnan(base[1]).any() and not torch.isnan(base[2]).any()


def test_backward_ignores_stale_gradient_outputs():
    """Every gradient element is written: outputs pre-filled with NaN give the same gradients as zero-filled ones."""
    s = ss.scene("stacks")
    P, H, W = s["means3D"].shape[0], s["H"], s["W"]
    R, color, radii, amap, geom, binning, image = raw_forward(s)
    t = _inputs(s)
    gi = torch.randn(3, H, W, device=DEV); gmap = torch.randn(9, H, W, device=DEV)
    cam = {k: torch.tensor(s[k], device=DEV) for k in ("bg", "viewmatrix", "projmatrix", "campos")}  # alive for the call
    outs = []
    for fillv in (0.0, float("nan")):
        g = [torch.full(sh, fillv, device=DEV) for sh in ((P, 3), (P, 1), (P, 3), (P, 3), (P, 16, 3), (P, 2), (P, 4))]
        f = lambda k: cam[k]
        rc = _lib.lib().gsr_surfel_backward(P, s["D"], 16, R, f("bg").data_ptr(), W, H, t["means3D"].data_ptr(),
                                            t["shs"].data_ptr(), t["scales"].data_ptr(), s["scale_modifier"],
                                            t["rotations"].data_ptr(), f("viewmatrix").data_ptr(),
                                            f("projmatrix").data_ptr(), f("campos").data_ptr(), geom.data_ptr(),
                                            binning.data_ptr(), image.data_ptr(), gi.data_ptr(), gmap.data_ptr(),
                                            *[x.data_ptr() for x in g], 0, torch.cuda.current_stream().cuda_stream)
        assert rc == 0, _lib.last_error()
        outs.append(g)
    for a, b in zip(*outs):
        assert not torch.isnan(b).any()
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)


# ---- end to end ---------------------------------------------------------------------------------------------------------
def _sphere_cameras(W=96, H=96):
    from gaustudio_b200.camera import orbit_cameras
    fov = math.radians(45.0)
    cams = []
    for el in (-65.0, -25.0, 15.0, 55.0, 85.0):
        cams += orbit_cameras(8, 2.0, el, W, H, fov, fov)
    return [c.to(torch.device(DEV)) for c in cams]


def _model_scene(model, cam):
    """The surfel scene dict (tests/surfel_scenes.py keys) of a point cloud seen by one camera."""
    a = lambda t: t.detach().cpu().numpy()
    W, H = int(cam.image_width), int(cam.image_height)
    return dict(W=W, H=H, D=model.active_sh_degree, scale_modifier=1.0, bg=np.zeros(3, np.float32),
                means3D=a(model.get_attribute("xyz")), scales=a(model.get_attribute("scale")),
                rotations=a(model.get_attribute("rot")), opacities=a(model.get_attribute("opacity")),
                shs=a(model.get_features), viewmatrix=a(cam.world_view_transform), projmatrix=a(cam.full_proj_transform),
                campos=a(cam.camera_center), tanfovx=math.tan(cam.FoVx * 0.5), tanfovy=math.tan(cam.FoVy * 0.5))


def test_2dgs_config_renderer_dict():
    from gaustudio_b200 import renderers
    r = renderers.make({"name": "surfel_renderer", "scaling_modifier": 1.0, "white_background": False,
                        "convert_SHs_python": False, "compute_cov3D_python": False, "debug": False})
    model = ss.sphere_model(n=2000)
    cam = _sphere_cameras(W=64, H=64)[5]
    pkg = r.render(cam, model)
    for k in ("render", "rendered_normal", "rendered_depth", "rendered_median_depth", "rendered_median_weight",
              "rendered_median_id", "viewspace_points", "visibility_filter", "rendered_final_opacity", "radii"):
        assert k in pkg, k
    assert pkg["rendered_median_id"].dtype == torch.int32
    # the dict is the float64 contract's maps, with the normal rotated to world space and depth = D / alpha
    s = _model_scene(model, cam)
    o = check_forward(s, what="sphere model")
    ok = (~o["flag"]).reshape(64, 64)
    a = pkg["rendered_final_opacity"][0].double()
    torch.testing.assert_close(a[ok], o["maps"][1].reshape(64, 64)[ok], rtol=0, atol=1e-4)
    V3 = torch.tensor(s["viewmatrix"], dtype=torch.float64, device=DEV)[:3, :3]
    nw = (o["maps"][2:5].T @ V3.T).T.reshape(3, 64, 64)
    torch.testing.assert_close(pkg["rendered_normal"].double()[:, ok], nw[:, ok], rtol=0, atol=1e-4)
    cov = ok & (a > 0.5)
    d = (o["maps"][0] / o["maps"][1]).reshape(64, 64)
    torch.testing.assert_close(pkg["rendered_depth"][0].double()[cov], d[cov], rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(pkg["rendered_median_id"][0][ok].long(), o["maps"][8].reshape(64, 64)[ok].long())


def test_extract_mesh_with_the_surfel_renderer():
    from gaustudio_b200 import mesh, renderers
    r = renderers.make("surfel_renderer")
    model = ss.sphere_model(n=6000, scale=0.02)
    vs = 0.02
    V, F = mesh.extract_mesh(r, model, _sphere_cameras(), voxel_size=vs, sdf_trunc=3 * vs, min_weight=1)
    assert F.shape[0] > 1000
    rad = V.norm(dim=1)
    assert float((rad - 0.5).abs().max()) < 1.5 * vs, float((rad - 0.5).abs().max())
    e = torch.cat([F[:, [0, 1]], F[:, [1, 2]], F[:, [2, 0]]]).sort(dim=1).values
    _, counts = torch.unique(e, dim=0, return_counts=True)
    assert bool((counts == 2).all()), "mesh is not closed"


def test_extract_pcd_with_the_surfel_renderer_and_no_renderer_syncs():
    from gaustudio_b200 import extract, renderers
    r = renderers.make("surfel_renderer")
    model = ss.sphere_model(n=4000, scale=0.025)
    cams = _sphere_cameras(W=80, H=80)
    with torch.no_grad():
        r.render(cams[0], model)  # the first view caches the background colour on the device
        # besides the forward's one count read (inside the library), rendering a view makes no torch-side
        # synchronisation, so the extraction loop is not held up by the renderer
        torch.cuda.set_sync_debug_mode("error")
        try:
            for cam in cams[:4]:
                r.render(cam, model)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    xyz, rgb, normals, _ = extract.extract_pcd(r, model, cams)
    assert xyz.shape[0] > 1000
    torch.testing.assert_close(xyz.norm(dim=1), torch.full_like(xyz[:, 0], 0.5), rtol=0, atol=1e-5)
    ok = ~torch.isnan(normals).any(1)
    assert ok.float().mean() > 0.5  # (the fusion leaves points whose views disagree without a normal)
    cosang = (normals[ok] * xyz[ok] / xyz[ok].norm(dim=1, keepdim=True)).sum(1).abs()
    # (the fused normals come from the filtered rendered depth, so silhouette pixels pull some of them off radial)
    assert float(cosang.median()) > math.cos(math.radians(2.0)), float(cosang.median())
    assert float((cosang > math.cos(math.radians(10.0))).float().mean()) > 0.9


def test_training_lowers_the_loss():
    from gaustudio_b200 import optimizers, renderers
    r = renderers.make("surfel_renderer")
    target_model = ss.sphere_model(n=1500, scale=0.04)
    cams = _sphere_cameras(W=64, H=64)[::4]
    with torch.no_grad():
        targets = [r.render(c, target_model)["render"] for c in cams]
    model = ss.sphere_model(n=1500, scale=0.04, seed=1, opacity=0.5)
    g = torch.Generator(device=DEV).manual_seed(0)
    model._xyz = model._xyz + 0.02 * torch.randn(model._xyz.shape, generator=g, device=DEV)
    model._f_dc = model._f_dc * 0.5
    model.requires_grad_(True)
    opt = optimizers.make({"name": "general", "model": model, "optimizer_name": "AdamW", "args": {"lr": 0.0, "eps": 1e-15},
                           "params": {"xyz": {"lr": 2e-4}, "opacity": {"lr": 0.05}, "f_dc": {"lr": 0.01},
                                      "scale": {"lr": 0.005}, "rot": {"lr": 0.001}}})
    losses = []
    for it in range(8):
        loss = sum((r.render(c, model)["render"] - t).abs().mean() for c, t in zip(cams, targets))
        loss.backward()
        opt.step()
        opt.zero_grad()
        losses.append(float(loss))
    assert all(b < a for a, b in zip(losses, losses[1:])), losses
