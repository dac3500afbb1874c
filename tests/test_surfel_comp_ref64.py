"""Pins the float64 surfel compositing reference (tests/surfel_comp_ref64.py) without a GPU.

* Against torch autograd of surfel_ref64.render on the same records as leaves (Tu, Tv, Tw, n_view, mean2D, opacity,
  rgb): the 18 closed-form sums agree to ~1e-10 of their magnitude, with every upstream channel alone and all of them
  together, on the small surfel scenes and on a tile whose list is longer than one 256-record batch.
* The forward maps agree with surfel_ref64.render, and the distortion with the pairwise sum.
* A float32 evaluation of the same closed forms lands well inside EPS * A (the bound can be met in float32), and
  A >= |S| componentwise.

Also the seeded surfel scenes the GPU comparison (tests/test_gpu_surfel_f64.py) adds to tests/surfel_scenes.py."""
import math

import numpy as np
import pytest
import torch

import surfel_comp_ref64 as R
import surfel_ref64 as ref
import surfel_scenes as ss
from test_gpu_compositing_f64 import _pix_to_u, _view_to_world

F32_MARGIN = 0.25
CHANNELS = {"image": None, "D": 0, "1-T": 1, "normal": (2, 3, 4), "median": 5, "distortion": 6}


# ---- scenes ---------------------------------------------------------------------------------------------------------
def view_scene(kind, W, H, seed, D=0):
    """Surfels placed in view space, in the format of surfel_scenes.scene.
    deep: > 600 low-opacity camera-facing surfels over tile (1, 1); saturating: opacities 0.99-1; thin: stacks of
    surfels whose depths differ by ~1e-3 z, with groups at identical positions; partial: any size; offscreen_large:
    centres off screen with rects of more than 32 tiles, plus 100:1 needles."""
    rng = np.random.RandomState(seed)
    cam = ss.camera(W, H)
    tx, ty = math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5)
    P = {"deep": 640, "saturating": 300, "thin": 240, "partial": max(60, W * H // 80), "offscreen_large": 300}[kind]
    z = rng.uniform(1.5, 4.0, P)
    u, v = rng.uniform(-1, 1, P) * tx, rng.uniform(-1, 1, P) * ty
    s = 0.03 * z[:, None] * np.exp(0.3 * rng.randn(P, 2))
    op = rng.uniform(0.1, 0.9, P)
    nrm = rng.randn(P, 3) * 0.4 + np.array([0.0, 0.0, -1.0])  # roughly facing the camera (view space)
    bg = np.array([0.2, 0.6, 0.4])
    if kind == "deep":
        z = rng.uniform(2.0, 3.0, P)
        u = _pix_to_u(24 + 2 * rng.randn(P), W, tx)
        v = _pix_to_u(24 + 2 * rng.randn(P), H, ty)
        s = 0.05 * z[:, None] * np.exp(0.1 * rng.randn(P, 2))
        op = rng.uniform(0.008, 0.014, P)
        nrm = rng.randn(P, 3) * 0.05 + np.array([0.0, 0.0, -1.0])
    elif kind == "saturating":
        op = rng.uniform(0.99, 1.0, P)
        s = 0.04 * z[:, None] * np.exp(0.3 * rng.randn(P, 2))
        bg = np.array([1.0, 1.0, 1.0])
    elif kind == "thin":
        # 24 stacks of 10: lateral jitter 1e-3, depths z0 (1 + 1e-3 k); every stack has a pair at one position
        n_st, per = 24, 10
        z0 = np.repeat(rng.uniform(2.5, 3.5, n_st), per)
        u = np.repeat(rng.uniform(-0.8, 0.8, n_st) * tx, per) + 1e-3 * rng.randn(P)
        v = np.repeat(rng.uniform(-0.8, 0.8, n_st) * ty, per) + 1e-3 * rng.randn(P)
        z = z0 * (1 + 1e-3 * np.tile(np.arange(per), n_st))
        z[1::per], u[1::per], v[1::per] = z[0::per], u[0::per], v[0::per]
        s = np.repeat(0.08 * z0[::per, None] * np.exp(0.2 * rng.randn(n_st, 2)), per, 0)
        op = rng.uniform(0.2, 0.6, P)
        nrm = np.repeat(rng.randn(n_st, 3) * 0.15 + np.array([0.0, 0.0, -1.0]), per, 0) + 0.01 * rng.randn(P, 3)
    elif kind == "offscreen_large":
        half = P // 2
        side = np.where(rng.rand(half) < 0.5, -1.0, 1.0)
        alongx = rng.rand(half) < 0.5
        u[:half] = np.where(alongx, side * tx * rng.uniform(1.05, 1.3, half), u[:half])
        v[:half] = np.where(~alongx, side * ty * rng.uniform(1.05, 1.3, half), v[:half])
        s[:half] = 0.35 * z[:half, None] * np.exp(0.2 * rng.randn(half, 2))
        op[:half] = rng.uniform(0.05, 0.3, half)
        s[half:, 1] = 0.003 * z[half:]
        s[half:, 0] = 0.3 * z[half:]
        nrm[half:] = rng.randn(P - half, 3)  # needles in every orientation
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    V3 = cam.world_view_transform.double().numpy()[:3, :3]
    n_world = nrm @ np.linalg.inv(V3)  # row vectors: n_view = n_world @ V3
    means = _view_to_world(cam, np.stack([u * z, v * z, z], 1))
    rot = ss.mat_to_quat(ss.frames_with_normal(n_world, rng))
    if kind == "thin":
        rot[1::10] = rot[0::10]
    sc = dict(case=kind, W=W, H=H, scale_modifier=1.0, bg=bg)
    return ss._finish(sc, means, s, rot, op, rng, cam, D=D)


# ---- records from the float64 projection (what a forward would leave in its geometry buffer) --------------------------
def records(s):
    """-> (rec dict of float32 tensors, radii) from surfel_ref64.project rounded to float32."""
    t = ref.scene_tensors(s, "cpu")
    g = ref.project(t["means3D"], t["scales"], t["rotations"], t["viewmatrix"], t["projmatrix"], s["W"], s["H"],
                    s["scale_modifier"])
    rgb = t["colors_precomp"] if t["colors_precomp"] is not None else ref.sh_colors(t["shs"], s["D"], t["means3D"],
                                                                                    t["campos"])
    f = lambda v: v.detach().float()
    rec = dict(mean2D=f(torch.stack([g["mx"], g["my"]], 1)), Tu=f(g["Tu"]), Tv=f(g["Tv"]), Tw=f(g["Tw"]),
               nv=f(g["nv"]), rgb=f(rgb), opacity=f(t["opacities"].reshape(-1)), depth=g["depth32"])
    _, live = ref.rects(g)
    radii = torch.where(live, g["radius"], torch.zeros_like(g["radius"])).long()
    return rec, radii


def render_on_records(rec, radii, s, leaves=True):
    """surfel_ref64.render with the records as (float64) leaves -> (render output, leaves dict)."""
    d = lambda k: rec[k].double().clone().requires_grad_(leaves)
    lv = {k: d(k) for k in ("Tu", "Tv", "Tw", "nv", "rgb", "opacity")}
    lv["mx"] = rec["mean2D"][:, 0].double().clone().requires_grad_(leaves)
    lv["my"] = rec["mean2D"][:, 1].double().clone().requires_grad_(leaves)
    r = radii.double()
    g = dict(P=r.numel(), W=s["W"], H=s["H"], Tu=lv["Tu"], Tv=lv["Tv"], Tw=lv["Tw"], nv=lv["nv"], mx=lv["mx"],
             my=lv["my"], radius=r, ok=radii > 0, rad_amb=torch.zeros_like(radii, dtype=torch.bool),
             depth32=rec["depth"].float())
    bg = torch.as_tensor(s["bg"], dtype=torch.float64)
    return ref.render(g, lv["opacity"], lv["rgb"], bg, trace=True), lv


def upstream(H, W, seed, only=None):
    """Random upstream (image [3,H,W], allmap [9,H,W], float32-representable); only: one channel group of CHANNELS."""
    g = torch.Generator().manual_seed(seed)
    img = torch.randn(3, H, W, generator=g).double()
    amap = torch.randn(9, H, W, generator=g).double()
    if only is not None:
        keep = CHANNELS[only]
        img = img if only == "image" else torch.zeros_like(img)
        mask = torch.zeros(9, 1, 1, dtype=torch.float64)
        if keep is not None:
            mask[list(keep) if isinstance(keep, tuple) else [keep]] = 1
        amap = amap * mask
    return img, amap


SCENES = {
    "random": lambda: ss.scene("random", D=1),
    "sphere": lambda: ss.scene("sphere", colors=True),
    "grazing": lambda: ss.scene("grazing", D=0),
    "near": lambda: ss.scene("near", D=0),
    "stacks": lambda: ss.scene("stacks", D=0, bg=(0.3, 0.5, 1.0)),
    "deep": lambda: view_scene("deep", 40, 36, 1),
}


@pytest.fixture(scope="module")
def prepared():
    cache = {}

    def get(name):
        if name not in cache:
            s = SCENES[name]()
            rec, radii = records(s)
            cache[name] = (s, rec, radii, R.SurfelCompositing(rec, radii, s["W"], s["H"], s["bg"]))
        return cache[name]
    return get


@pytest.mark.parametrize("name", list(SCENES))
def test_sums_match_autograd_of_the_contract(prepared, name):
    s, rec, radii, ref64 = prepared(name)
    H, W = s["H"], s["W"]
    if name == "deep":
        assert int(ref64.last.max()) > 256 and int(ref64.n_contrib.max()) > 256
    worst = 0.0
    for i, only in enumerate([None] + list(CHANNELS)):
        img, amap = ref64.masked(*upstream(H, W, 10 + i, only))
        out, lv = render_on_records(rec, radii, s)
        keep = (~out["flag"]).double().reshape(H, W)
        img, amap = img * keep, amap * keep
        loss = (out["image"] * img.reshape(3, -1)).sum() + (out["maps"][:7] * amap[:7].reshape(7, -1)).sum()
        loss.backward()
        S, A = ref64.sums(img, amap, drop_flagged=False)
        assert (A >= S.abs()).all(), (name, only)
        got = torch.cat([lv["mx"].grad[:, None], lv["my"].grad[:, None], lv["Tu"].grad, lv["Tv"].grad, lv["Tw"].grad,
                         lv["nv"].grad, lv["opacity"].grad[:, None], lv["rgb"].grad], 1)
        r, gi, c = R.worst_ratio(got, S, A, eps=1e-10)
        assert r <= 1, f"{name} / {only}: Gaussian {gi} {R.NAMES[c]}: autograd {float(got[gi, c]):.12g} " \
                       f"closed form {float(S[gi, c]):.12g}"
        worst = max(worst, r)
        if only is not None:
            assert ref64.reached.any(), (name, only)
    print(f"\n{name}: worst |closed form - autograd| / (1e-10 A) = {worst:.3g}")


@pytest.mark.parametrize("name", list(SCENES))
def test_forward_maps_match_the_contract(prepared, name):
    s, rec, radii, ref64 = prepared(name)
    out, _ = render_on_records(rec, radii, s, leaves=False)
    ok = ~out["flag"] & ~ref64.flag & ~ref64.flag_median
    assert ok.float().mean() > 0.5, name
    mp = ref64.maps()
    close = lambda a, b: float((a - b).abs().max()) if a.numel() else 0.0
    assert close(mp["image"][0][:, ok], out["image"][:, ok].detach()) < 1e-12
    for c, key in ((0, "D"), (1, "1-T"), (5, "median depth"), (6, "distortion")):
        assert close(mp[key][0][ok], out["maps"][c][ok].detach()) < 1e-12, (name, key)
        assert (mp[key][1] >= mp[key][0].abs()).all()
    assert close(mp["normal"][0][:, ok], out["maps"][2:5][:, ok].detach()) < 1e-12
    assert torch.equal(mp["median id"][ok].double().clamp(min=0), out["maps"][8][ok].detach()), name
    # the distortion is the pairwise sum over the pixel's blended splats
    wts, dep = out["weights"], out["depths"]
    for p in ok.nonzero().flatten()[:: max(1, int(ok.sum()) // 40)].tolist():
        wp = wts[:, p]
        sel = wp > 0
        pw = ref.pairwise_distortion(wp[sel].tolist(), [ref.m_of(float(zz)) for zz in dep[:, p][sel]])
        assert abs(float(mp["distortion"][0][p]) - pw) <= 1e-12 * (1 + abs(pw)), (name, p)


@pytest.mark.parametrize("name", list(SCENES))
def test_float32_closed_forms_within_the_bound(prepared, name):
    s, rec, radii, ref64 = prepared(name)
    r32 = R.SurfelCompositing(rec, radii, s["W"], s["H"], s["bg"], dtype=torch.float32)
    worst = {}
    for i, only in enumerate([None, "image", "D", "normal", "median", "distortion"]):
        img, amap = ref64.masked(*upstream(s["H"], s["W"], 30 + i, only))
        S, A = ref64.sums(img, amap, drop_flagged=False)
        S32, _ = r32.sums(img.float(), amap.float(), drop_flagged=False)
        worst[only] = R.worst_ratio(S32, S, A)[0]
    mp, mp32 = ref64.maps(), r32.maps()
    keep = ~ref64.flag
    for k in ("image", "D", "1-T", "normal", "median depth", "distortion"):
        v, a = mp[k]
        worst[k] = R.worst_ratio(mp32[k][0][..., keep].reshape(-1), v[..., keep].reshape(-1),
                                 a[..., keep].reshape(-1))[0]
    print(f"\n{name}: float32 / bound " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))
    assert max(worst.values()) <= F32_MARGIN, (name, worst)


def test_scene_builders():
    """The extra scenes have what they are there for (from the float64 projection; the GPU test asserts the same on
    the GPU's records)."""
    s = view_scene("thin", 64, 48, 5)
    rec, radii = records(s)
    d = rec["depth"][radii > 0]
    assert len(d) - len(torch.unique(d)) >= 20  # identical positions
    r = R.SurfelCompositing(rec, radii, 64, 48, s["bg"])
    assert r.covered.sum() > 500


# ---- what the error model assumes of the compiled kernels ------------------------------------------------------------
def _sass_of_surfel_kernels():
    """SASS of gsr_surfel.cu built with the library's flags -> {kernel name fragment: [instruction text]}."""
    import os
    import re
    import subprocess
    import tempfile
    from gaustudio_b200 import build as b
    flags = [f for f in b.FLAGS if f not in ("-Xptxas", "-v", "-Xcompiler", "-fPIC")]
    with tempfile.TemporaryDirectory() as tmp:
        cubin = os.path.join(tmp, "surfel.cubin")
        subprocess.run([b.NVCC, *flags, "-cubin", "-o", cubin, os.path.join(b.CSRC, "gsr_surfel.cu")], check=True,
                       capture_output=True)
        sass = subprocess.run([os.path.join(os.path.dirname(b.NVCC), "cuobjdump"), "-sass", cubin], check=True,
                              capture_output=True, text=True).stdout
    out, cur = {}, None
    for line in sass.splitlines():
        if "Function :" in line:
            cur = next((k for k in ("k_surfel_render_fwd", "k_surfel_render_bwd") if k in line), None)
            if cur:
                out[cur] = []
        elif cur:
            m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", line)
            if m:
                out[cur].append(m.group(1))
    return out


@pytest.mark.skipif(not __import__("os").path.exists(__import__("gaustudio_b200.build").build.NVCC),
                    reason="nvcc not available")
def test_ray_splat_rows_are_single_ffmas():
    """The reference's error model takes k = x Tw - Tu and l = y Tw - Tv as one FFMA per component (exact product,
    one rounding: |dk| <= u |k|).  A separate multiply and subtract would cost u |x Tw|, about a thousand times |k|
    at 1080p, and widen every bound that rests on the ray-splat intersection.  In both compositing kernels, right after
    a record is read from shared memory, the six components must be FFMAs with a negated addend, three on the register
    holding the pixel's x and three on the one holding its y."""
    import re
    ffma = re.compile(r"FFMA R\d+, (R\d+)(?:\.reuse)?, R\d+(?:\.reuse)?, -R\d+$")
    for name, ins in _sass_of_surfel_kernels().items():
        first = next(i for i, t in enumerate(ins) if t.startswith("LDS.128"))
        window = ins[first:first + 40]
        srcs = [m.group(1) for m in (ffma.match(t) for t in window) if m]
        coords = [r for r in set(srcs) if srcs.count(r) >= 3]
        assert len(coords) == 2, (name, window)
        # and no plain multiply of a pixel coordinate there (what an uncontracted x * Tw would be)
        assert not any(t.startswith("FMUL") and re.search(rf"\b{c}\b", t) for t in window for c in coords), (name, window)
