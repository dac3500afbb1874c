"""-m gpu: the compositing backward (k_render_bwd) against the float64 reference of tests/comp_ref64.py.

A real forward fills the state buffers; the production gsr_backward then runs on chosen upstream images, and the
accumulator it leaves in the geometry buffer (gsr_debug_accumulator) is compared with the reference's ten sums: every
component of every Gaussian within EPS * A (comp_ref64's error model), no outlier budget.  Pixels where a decision of
the reference lies within float32 rounding of its threshold get zero upstream on both sides (only the median-depth
image where the ambiguous decision is the median crossing).

Scenes: A-D, a tile deeper than the ring (> NSTAGE * RB = 512 contributors), near-opaque splats (0.99 clamp, early
ends at different depths in one 8x4 block), partial tiles (13x7, 250x170), off-screen centres and thin rotated
ellipses, equal depths.  Upstream: random on all four images, each image alone, one pixel (tile corner, last row and
column), one 8x4 block, a checkerboard of signs, magnitudes from 1e-3 to 1e3.  Exact checks on top of the bound:
Gaussians no pixel with upstream reaches are all-zero, slots 10-11 are zero, an image alone moves only its
components, and the median-depth gradient lands exactly on the forward's median Gaussians.  Variants: the three tile
orders, two pixels per lane (GSR_BWD_NSUB=2) and the one-stage-ring build (when it has been built)."""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import comp_ref64 as R
import scenes

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STRESS = os.path.join(ROOT, "gaustudio_b200", "libgsr_b200_stress.so")
MAX_FLAGGED = 0.01  # of the covered pixels


def _view_to_world(cam, pv):
    V = cam.world_view_transform.double().numpy()
    return (pv - V[3, :3]) @ np.linalg.inv(V[:3, :3])


def _pix_to_u(x, W, tan):
    """view-space x / z of pixel column x (inverse of the NDC -> pixel map)"""
    return ((2 * x + 1) / W - 1) * tan


def view_scene(kind, W, H, seed):
    """Gaussians placed in view space, shs of degree 0, in the format of scenes.scene."""
    rng = np.random.RandomState(seed)
    cam = scenes.camera(W, H, 50.0)
    tx, ty = math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5)
    P = {"deep": 700, "saturating": 400, "partial": max(60, W * H // 60), "offscreen_thin": 600, "equal": 400,
         "wide": 1200}[kind]
    z = rng.uniform(1.5, 4.0, P)
    u, v = rng.uniform(-1, 1, P) * tx, rng.uniform(-1, 1, P) * ty
    s = 0.025 * z[:, None] * np.exp(0.3 * rng.randn(P, 3))
    op = rng.uniform(0.05, 0.95, P)
    bg = np.array([0.2, 0.6, 0.4])
    if kind == "deep":
        # low-opacity splats ~10 px wide around the centre of tile (1, 1): > 512 contributors, T stays above 1e-4
        z = rng.uniform(2.0, 3.0, P)
        u = _pix_to_u(24 + 3 * rng.randn(P), W, tx)
        v = _pix_to_u(24 + 3 * rng.randn(P), H, ty)
        s = 0.2 * z[:, None] * np.exp(0.1 * rng.randn(P, 3))
        op = rng.uniform(0.008, 0.016, P)
    elif kind == "saturating":
        op = np.where(rng.rand(P) < 0.5, rng.uniform(0.995, 1.0, P), rng.uniform(0.85, 0.995, P))
        s = 0.05 * z[:, None] * np.exp(0.3 * rng.randn(P, 3))
        bg = np.array([1.0, 1.0, 1.0])
    elif kind == "wide":
        # small splats (sigma ~ 2-5 px) all over an image of several tile-scan rounds (8192 tiles each)
        s = 0.0018 * z[:, None] * np.exp(0.3 * rng.randn(P, 3))
        # and a few wider ones on the centre of the image, where the one-block upstream pattern lies
        u[:8], v[:8] = _pix_to_u(W / 2 + 4 * rng.randn(8), W, tx), _pix_to_u(H / 2 + 2 * rng.randn(8), H, ty)
        s[:8] *= 3
    elif kind == "offscreen_thin":
        half = P // 2
        # centres beyond the image edges (inside the lateral clamp), wide enough to reach the screen
        side = np.where(rng.rand(half) < 0.5, -1.0, 1.0)
        alongx = rng.rand(half) < 0.5
        u[:half] = np.where(alongx, side * tx * rng.uniform(1.03, 1.25, half), u[:half])
        v[:half] = np.where(~alongx, side * ty * rng.uniform(1.05, 1.25, half), v[:half])
        s[:half] = 0.12 * z[:half, None] * np.exp(0.2 * rng.randn(half, 3))
        # the other half: needles, 100 : 1, in every orientation
        s[half:] = 0.004 * z[half:, None] * np.ones((P - half, 3))
        s[half:, 0] = 0.25 * z[half:]
    q = rng.randn(P, 4)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    means = _view_to_world(cam, np.stack([u * z, v * z, z], 1))
    if kind == "equal":
        means[1::4] = means[0::4][: len(means[1::4])]  # groups of Gaussians at one position share their depth exactly
        means[2::4] = means[0::4][: len(means[2::4])]
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    return dict(case=kind, W=W, H=H, D=0, scale_modifier=1.0, bg=f32(bg), means3D=f32(means), scales=f32(s),
                rotations=f32(q), opacities=f32(op[:, None]), shs=f32(rng.randn(P, 1, 3)),
                viewmatrix=cam.world_view_transform.numpy(), projmatrix=cam.full_proj_transform.numpy(),
                campos=cam.camera_center.numpy(), tanfovx=tx, tanfovy=ty)


SCENES = {
    "A": lambda: scenes.scene("A"), "B": lambda: scenes.scene("B"), "C": lambda: scenes.scene("C"),
    "D": lambda: scenes.scene("D"),
    "deep": lambda: view_scene("deep", 64, 48, 1),
    "saturating": lambda: view_scene("saturating", 64, 48, 2),
    "partial13x7": lambda: view_scene("partial", 13, 7, 3),
    "partial250x170": lambda: view_scene("partial", 250, 170, 4),
    "offscreen_thin": lambda: view_scene("offscreen_thin", 64, 48, 5),
    "equal": lambda: view_scene("equal", 64, 48, 6),
    "wide3840x2160": lambda: view_scene("wide", 3840, 2160, 7),   # four rounds, the last one partial
    "wide2561x1441": lambda: view_scene("wide", 2561, 1441, 8),   # two rounds, partial tiles on both edges
}


class Frame:
    """One forward on the GPU, its state buffers kept alive, and the reference built from its exported state."""

    def __init__(self, s, dev):
        from gaustudio_b200 import _C
        self.s, self.dev, self.W, self.H = s, dev, s["W"], s["H"]
        e = torch.Tensor([])
        d = lambda k: torch.as_tensor(s[k]).to(dev).contiguous() if s.get(k) is not None else e
        self.t = {k: d(k) for k in ("means3D", "colors_precomp", "opacities", "scales", "rotations", "cov3D_precomp",
                                    "shs")}
        self.bg = torch.as_tensor(s["bg"], dtype=torch.float32).to(dev)
        self.cam = tuple(torch.as_tensor(np.asarray(s[k], dtype=np.float32)).to(dev).contiguous()
                         for k in ("viewmatrix", "projmatrix", "campos"))
        t = self.t
        (self.R, _, _, median, _, self.radii, self.gb, self.bb, self.ib) = _C.rasterize_gaussians(
            self.bg, t["means3D"], t["colors_precomp"], t["opacities"], t["scales"], t["rotations"],
            s["scale_modifier"], t["cov3D_precomp"], self.cam[0], self.cam[1], s["tanfovx"], s["tanfovy"], self.H,
            self.W, t["shs"], s["D"], self.cam[2], False, False)
        self.P = self.radii.numel()
        ex = _C.debug_export(self.P, self.W, self.H, self.R, self.gb, self.bb, self.ib)
        self.ex = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in ex.items()}
        self.median_w = median[1].cpu().reshape(-1)
        self.median_id = median[2].cpu().reshape(-1).long()
        rgb = s["colors_precomp"] if s.get("colors_precomp") is not None else self.ex["rgb"]
        self.ref = R.Compositing(self.ex["means2D"], self.ex["conic_opacity"], rgb, self.ex["depths"],
                                 self.radii.cpu(), self.W, self.H, s["bg"])

    def backward(self, up):
        """gsr_backward on the upstream images `up` (dpix [3,H,W], ddepth, dmedian (channel 0), dopacity [H,W]); ->
        the accumulator [P,12] it left in the geometry buffer."""
        from gaustudio_b200 import _C
        s, t, dev, H, W = self.s, self.t, self.dev, self.H, self.W
        dm = torch.zeros(3, H, W)
        dm[0] = up[2]
        gpu = [up[0].float().to(dev), up[1].float().reshape(1, H, W).to(dev), dm.to(dev),
               up[3].float().reshape(1, H, W).to(dev)]
        _C.rasterize_gaussians_backward(self.bg, t["means3D"], self.radii, t["colors_precomp"], t["scales"],
                                        t["rotations"], s["scale_modifier"], t["cov3D_precomp"], self.cam[0],
                                        self.cam[1], s["tanfovx"], s["tanfovy"], *gpu, t["shs"], s["D"], self.cam[2],
                                        self.gb, self.R, self.bb, self.ib, False)
        acc = _C.debug_accumulator(self.P, self.gb)
        torch.cuda.synchronize()
        return acc.cpu()

    def tile_maxc(self):
        """largest n_contrib of each tile (what bounds the backward's traversal), from the GPU's own state"""
        W, H = self.W, self.H
        nc = self.ex["n_contrib"].reshape(H, W).numpy()
        gx, gy = (W + 15) // 16, (H + 15) // 16
        return np.array([nc[ty * 16:(ty + 1) * 16, tx * 16:(tx + 1) * 16].max()
                         for ty in range(gy) for tx in range(gx)])


def patterns(W, H, seed):
    """name -> (dpix [3,H,W], ddepth [H,W], dmedian [H,W], dopacity [H,W]), float32-representable."""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *sh: torch.randn(*sh, generator=g)
    z = lambda *sh: torch.zeros(*sh)
    out = {"random": (rn(3, H, W), rn(H, W), rn(H, W), rn(H, W)),
           "color": (rn(3, H, W), z(H, W), z(H, W), z(H, W)),
           "depth": (z(3, H, W), rn(H, W), z(H, W), z(H, W)),
           "median": (z(3, H, W), z(H, W), 0.5 + torch.rand(H, W, generator=g), z(H, W)),
           "opacity": (z(3, H, W), z(H, W), z(H, W), rn(H, W))}
    for name, (x, y) in (("pixel_corner", (16, 16) if W > 16 and H > 16 else (0, 0)), ("pixel_last", (W - 1, H - 1))):
        m = z(H, W)
        m[y, x] = 1
        out[name] = (rn(3, H, W) * m, rn(H, W) * m, rn(H, W) * m, rn(H, W) * m)
    m = z(H, W)
    bx, by = (W // 2) // 8 * 8, (H // 2) // 4 * 4  # the 8x4 block at the centre of the image
    m[by:by + 4, bx:bx + 8] = 1
    out["block"] = (rn(3, H, W) * m, rn(H, W) * m, rn(H, W) * m, rn(H, W) * m)
    yy, xx = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    chk = ((xx + yy) % 2 * 2 - 1).float()
    out["checker"] = (rn(3, H, W).abs() * chk, rn(H, W).abs() * chk, rn(H, W).abs() * chk, rn(H, W).abs() * chk)
    mag = lambda *sh: torch.sign(rn(*sh)) * 10.0 ** (6 * torch.rand(*sh, generator=g) - 3)
    out["spread"] = (mag(3, H, W), mag(H, W), mag(H, W), mag(H, W))
    return {k: tuple(x.float() for x in v) for k, v in out.items()}


def check(fr, name, up, acc, ref):
    """The bound and the exact structural checks for one backward; -> worst error / bound."""
    S, A = ref
    what = f"{fr.s['case']} / {name}"
    assert torch.isfinite(acc).all(), what
    assert not acc[:, 10:].any(), f"{what}: slots 10-11 not zero"
    dead = ~fr.ref.reached
    assert not acc[dead].any(), f"{what}: a Gaussian no pixel with upstream reaches has a non-zero sum " \
                                f"(#{int((acc[dead] != 0).any(1).nonzero()[0, 0])})"
    r, i, c = R.worst_ratio(acc[:, :10], S[:, :10], A[:, :10])
    assert r <= 1, f"{what}: Gaussian {i} component {R.LOG_NAMES[c]}: gpu {float(acc[i, c]):.9g} ref " \
                   f"{float(S[i, c]):.9g} at {r:.3g} x the bound ({float(R.EPS * A[i, c]):.3g})"
    if name == "color":
        assert not acc[:, 3].any(), what
    if name == "depth":
        assert not acc[:, 0:3].any(), what
    if name == "opacity":
        assert not acc[:, 0:4].any(), what
    if name == "median":
        assert not acc[:, [0, 1, 2, 4, 5, 6, 7, 8, 9]].any(), what
        keep = (fr.median_w > 0) & (up[2].reshape(-1) != 0)  # `up` is masked: ambiguous pixels have none
        want = torch.zeros(fr.P, dtype=torch.bool)
        want[fr.median_id[keep]] = True
        assert torch.equal(acc[:, 3] != 0, want), f"{what}: median gradient not on the forward's median Gaussians"
    return r


def run_scene(key, dev, orders=(1, 0, 2), names=None):
    """All upstream patterns on one scene (default tile order), then the random pattern under every tile order.
    -> (worst error / bound, flagged fraction)."""
    from gaustudio_b200 import _C
    fr = Frame(SCENES[key](), dev)
    st = fr.ref.stats()
    assert st["frac"] < MAX_FLAGGED, (key, st)
    # the forward's median Gaussian is the reference's wherever the decision is not ambiguous
    sure = ~fr.ref.flag & ~fr.ref.flag_median
    assert torch.equal((fr.median_w > 0)[sure], (fr.ref.median >= 0)[sure]), key
    m = sure & (fr.median_w > 0)
    assert torch.equal(fr.median_id[m], fr.ref.median[m]), key
    pats = patterns(fr.W, fr.H, sum(map(ord, key)))
    worst = 0.0
    prev = _C.set_tile_order(orders[0])
    try:
        for name, up in pats.items():
            if names is not None and name not in names:
                continue
            up = fr.ref.masked(*up)
            ref = fr.ref.sums(*up)
            assert bool(fr.ref.reached.any()) or name.startswith("pixel"), (key, name)
            worst = max(worst, check(fr, name, up, fr.backward(up), ref))
            if name == "random":
                for o in orders[1:]:
                    _C.set_tile_order(o)
                    worst = max(worst, check(fr, f"{name} tile order {o}", up, fr.backward(up), ref))
                _C.set_tile_order(orders[0])
    finally:
        _C.set_tile_order(prev)
    return fr, worst, st


@pytest.mark.parametrize("key", list(SCENES))
def test_accumulator_matches_f64_reference(key):
    dev = torch.device("cuda")
    fr, worst, st = run_scene(key, dev)
    ref = fr.ref
    # what the scene is there for
    if key == "deep":
        mc = fr.tile_maxc()
        deep = mc[mc > 512]
        assert len(deep) and (deep % 32 != 0).any(), mc
        assert int(ref.n_contrib.max()) > 512 and float(ref.final_T[ref.n_contrib > 512].min()) > 1e-4
    if key == "saturating":
        clamped = sum(int((tl["oG"] > R.ALPHA_MAX).sum()) for tl in ref.tiles)
        assert clamped >= 20, clamped
        # pixels of one 8x4 block end at different depths
        W, H = fr.W, fr.H
        ended = ref.ended.reshape(H, W)
        nc = ref.n_contrib.reshape(H, W)
        mixed = 0
        for by in range(0, H - 3, 4):
            for bx in range(0, W - 7, 8):
                e, n = ended[by:by + 4, bx:bx + 8], nc[by:by + 4, bx:bx + 8]
                mixed += int(e.sum() >= 2 and len(set(n[e].tolist())) > 1)
        assert mixed >= 10, mixed
    if key.startswith("partial"):
        cov = ref.covered.reshape(fr.H, fr.W)
        assert cov[-1].any() and cov[:, -1].any() and cov[-1, -1]
        assert fr.W % 16 and fr.H % 16 and fr.H % 4
    if key == "offscreen_thin":
        m2 = fr.ex["means2D"]
        off = (m2[:, 0] < 0) | (m2[:, 0] >= fr.W) | (m2[:, 1] < 0) | (m2[:, 1] >= fr.H)
        S, _ = ref.sums(*patterns(fr.W, fr.H, 0)["random"])
        live = (S[:, :10] != 0).any(1)
        assert int((off & live).sum()) >= 20
        co = fr.ex["conic_opacity"].double()
        tr, det = co[:, 0] + co[:, 2], co[:, 0] * co[:, 2] - co[:, 1] ** 2
        disc = torch.sqrt((tr * tr / 4 - det).clamp(min=0))
        ratio = (tr / 2 + disc) / (tr / 2 - disc).clamp(min=1e-30)
        assert int((live & (ratio > 100) & (co[:, 1].abs() > 0.2 * co[:, 0].abs())).sum()) >= 20
    if key.startswith("wide"):
        # Gaussians reached by the upstream in every round of the tile scan
        gx = (fr.W + 15) // 16
        T = gx * ((fr.H + 15) // 16)
        cov = ref.covered.reshape(fr.H, fr.W).nonzero()
        hit = set(((cov[:, 0] // 16) * gx + cov[:, 1] // 16).div(8192, rounding_mode="floor").tolist())
        assert T > 8192 and hit == set(range((T + 8191) // 8192)), (T, hit)
    if key == "equal":
        d = fr.ex["depths"][fr.radii.cpu() > 0]
        assert len(d) - len(torch.unique(d)) >= 50
    print(f"\n{key}: worst error / bound {worst:.3g}; of {st['covered']} covered pixels {100 * st['frac']:.2f} % "
          f"flagged, {100 * st['median_frac']:.2f} % with an ambiguous median")


CHILD = r'''
import json, sys, torch
sys.path[:0] = [".", "tests"]
import test_gpu_compositing_f64 as T
out = {}
for key in T.SCENES:
    fr, worst, st = T.run_scene(key, torch.device("cuda"), orders=(1,), names=("random", "checker", "median"))
    out[key] = worst
print("RESULT" + json.dumps(out))
'''


def _child(lib=None, **env_extra):
    env = dict(os.environ)
    env.pop("GSR_BWD_NSUB", None)
    env.pop("GSR_LIB", None)
    if lib:
        env["GSR_LIB"] = lib
    env.update(env_extra)
    r = subprocess.run([sys.executable, "-c", CHILD], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    out = json.loads([l for l in r.stdout.splitlines() if l.startswith("RESULT")][-1][6:])
    print("\n" + ", ".join(f"{k} {v:.3g}" for k, v in out.items()))
    return out


def test_two_pixels_per_lane_against_f64_reference():
    """GSR_BWD_NSUB=2 (read once per process, hence the child process): the same bound on every scene."""
    _child(GSR_BWD_NSUB="2")


def test_one_stage_ring_against_f64_reference():
    if not os.path.exists(STRESS):
        pytest.skip("stress variant not built "
                    "(python -c 'from gaustudio_b200 import build; build.build_stress_variant()')")
    _child(STRESS)
