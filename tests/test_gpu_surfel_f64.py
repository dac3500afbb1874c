"""-m gpu: the surfel backward, stage by stage, and the surfel forward per pixel, against float64 references.

A real forward (_C.rasterize_surfels) fills the state buffers; the production gsr_surfel_backward then runs on chosen
upstreams.  The records and the accumulator are read from the geometry buffer at the layout of carve_sgeom
(`geom_views`, pinned to gsr_surfel_geometry_bytes).

* k_surfel_render_bwd: the accumulator against tests/surfel_comp_ref64.py, built from the GPU's own records: every one
  of the 18 components of every Gaussian within EPS * A, no outlier budget.  Exact structural checks on top: slots
  18-19 zero, Gaussians no pixel with upstream reaches all-zero, each channel alone moves only its components, the
  median gradient lands exactly on the forward's median ids, channels 7-8 move nothing.
* k_surfel_render_fwd: image, D, 1 - T, normal, median depth and distortion per pixel within their bounds, the median
  id exact, on unflagged pixels.
* k_surfel_project_bwd: the GPU's accumulator, in float64, pushed through autograd of surfel_ref64.project and sh_colors
  (EPS_P * A_P, see `check_projection`), exact zeros where they are due.

Scenes: tests/surfel_scenes.py (random, sphere, grazing, near, stacks, plane) and the view-space scenes of
tests/test_surfel_comp_ref64.py (deep: a tile list > 512 entries; saturating: opacities 0.99-1; thin: depths 1e-3 z
apart with identical positions; partial 13x7 and 250x170; offscreen_large: rects of > 32 tiles and 100:1 needles), and
100k surfels at 1920x1080 with the upstream confined to sampled tiles."""

import numpy as np
import pytest
import torch

import surfel_comp_ref64 as R
import surfel_ref64 as ref
import surfel_scenes as ss
from test_surfel_comp_ref64 import view_scene

pytestmark = pytest.mark.gpu
DEV = "cuda"
MAX_FLAGGED = 0.01      # of the covered pixels
MAX_FLAGGED_GRAZING = 0.05
EPS_P = 16 * R.U


# ---- the geometry buffer --------------------------------------------------------------------------------------------
def geom_layout(P):
    """Byte offsets of carve_sgeom's arrays from the buffer's 256-aligned base; 'end': one past the accumulator."""
    a256 = lambda v: (v + 255) // 256 * 256
    off, p = {}, 0
    for name, nbytes in (("recA", P * 48), ("recB", P * 32), ("rect", P * 8), ("tile_mask", P * 4), ("radii", P * 4),
                         ("clamped", P), ("grad", P * 80)):
        p = a256(p)
        off[name] = p
        p += nbytes
    off["end"] = p
    return off


def geom_views(geom, P):
    """Views of the surfel geometry buffer: recA [P,12] float, recB [P,8], rect [P,2] int32, radii [P], clamped [P]
    uint8, grad [P,20] float (the compositing-backward accumulator)."""
    base = (-geom.data_ptr()) % 256
    off = geom_layout(P)
    v = lambda name, n, dt: geom[base + off[name]:base + off[name] + n * torch.tensor([], dtype=dt).element_size()]\
        .view(dt)
    return dict(recA=v("recA", P * 12, torch.float32).view(P, 12), recB=v("recB", P * 8, torch.float32).view(P, 8),
                rect=v("rect", P * 2, torch.int32).view(P, 2), radii=v("radii", P, torch.int32),
                clamped=geom[base + off["clamped"]:base + off["clamped"] + P],
                grad=v("grad", P * 20, torch.float32).view(P, 20))


def test_geom_layout_matches_the_library():
    from gaustudio_b200 import _lib
    L = _lib.lib()
    for P in (0, 1, 7, 100, 4097, 100000):
        assert geom_layout(P)["end"] + 512 == L.gsr_surfel_geometry_bytes(P), P


# ---- one forward, its buffers kept -----------------------------------------------------------------------------------
class Frame:
    def __init__(self, s, tiles=None):
        from gaustudio_b200 import _C
        self.s, self.W, self.H = s, s["W"], s["H"]
        f = lambda k: torch.tensor(np.asarray(s[k], dtype=np.float32), device=DEV)
        e = torch.empty(0, device=DEV)
        self.t = dict(means3D=f("means3D"), opacities=f("opacities"), scales=f("scales"), rotations=f("rotations"),
                      colors=f("colors_precomp") if "colors_precomp" in s else e, shs=f("shs") if "shs" in s else e)
        self.cam = dict(bg=f("bg"), view=f("viewmatrix"), proj=f("projmatrix"), campos=f("campos"))
        t, c = self.t, self.cam
        (self.R, color, radii, allmap, self.gb, self.bb, self.ib) = _C.rasterize_surfels(
            c["bg"], t["means3D"], t["colors"], t["opacities"], t["scales"], t["rotations"], s["scale_modifier"],
            c["view"], c["proj"], s["tanfovx"], s["tanfovy"], self.H, self.W, t["shs"], s["D"], c["campos"], False, False)
        torch.cuda.synchronize()
        self.P = t["means3D"].shape[0]
        self.radii = radii
        self.color, self.allmap = color.cpu().double(), allmap.cpu().double()
        v = geom_views(self.gb, self.P)
        self.rec = R.unpack_records(v["recA"].cpu(), v["recB"].cpu())
        self.clamped = v["clamped"].cpu()
        assert torch.equal(v["radii"].cpu(), radii.cpu())
        self.ref = R.SurfelCompositing(self.rec, radii.cpu(), self.W, self.H, s["bg"], tiles)

    def backward(self, img, amap):
        """gsr_surfel_backward on img [3,H,W], amap [9,H,W] -> (accumulator [P,20] float64, input gradients)."""
        from gaustudio_b200 import _C
        s, t, c = self.s, self.t, self.cam
        gi, gm = img.float().contiguous().to(DEV), amap.float().contiguous().to(DEV)
        out = _C.rasterize_surfels_backward(c["bg"], t["means3D"], self.radii, t["colors"], t["scales"],
                                            t["rotations"], s["scale_modifier"], c["view"], c["proj"], s["tanfovx"],
                                            s["tanfovy"], gi, gm, t["shs"], s["D"], c["campos"], self.gb, self.R,
                                            self.bb, self.ib, False)
        acc = geom_views(self.gb, self.P)["grad"].cpu().double()
        names = ("means2D", "colors", "opacity", "means3D", "shs", "scales", "rotations")
        return acc, {k: v.cpu().double() for k, v in zip(names, out)}


def patterns(W, H, seed, region=None):
    """name -> (img [3,H,W], amap [9,H,W]), float32-representable; region [H,W] bool confines every pattern."""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *sh: torch.randn(*sh, generator=g)
    one = lambda chans: (torch.zeros(3, H, W), torch.zeros(9, H, W).index_copy(0, torch.tensor(chans), rn(len(chans), H, W)))
    out = {"random": (rn(3, H, W), torch.cat([rn(7, H, W), rn(2, H, W)])),
           "image": (rn(3, H, W), torch.zeros(9, H, W)),
           "D": one([0]), "1-T": one([1]), "normal": one([2, 3, 4]), "median": one([5]), "distortion": one([6]),
           "channels 7-8": one([7, 8])}
    for name, (x, y) in (("pixel corner", (16, 16) if W > 16 and H > 16 else (0, 0)), ("pixel last", (W - 1, H - 1))):
        m = torch.zeros(H, W)
        m[y, x] = 1
        out[name] = (rn(3, H, W) * m, rn(9, H, W) * m)
    m = torch.zeros(H, W)
    ty, tx = ((H - 1) // 16) // 2, ((W - 1) // 16) // 2
    m[ty * 16:ty * 16 + 16, tx * 16:tx * 16 + 16] = 1
    out["tile"] = (rn(3, H, W) * m, rn(9, H, W) * m)
    yy, xx = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    chk = ((xx + yy) % 2 * 2 - 1).float()
    out["checker"] = (rn(3, H, W).abs() * chk, rn(9, H, W).abs() * chk)
    mag = lambda *sh: torch.sign(rn(*sh)) * 10.0 ** (6 * torch.rand(*sh, generator=g) - 3)
    out["spread"] = (mag(3, H, W), mag(9, H, W))
    if region is not None:
        out = {k: (a * region, b * region) for k, (a, b) in out.items()}
    return {k: (a.float().double(), b.float().double()) for k, (a, b) in out.items()}


SLOTS = dict(mean2D=[0, 1], T=list(range(2, 11)), normal=[11, 12, 13], opacity=[14], rgb=[15, 16, 17])


def check_backward(fr, name, up, acc):
    """Bound and structure of one accumulator -> (worst error / bound, S, A)."""
    what = f"{fr.s['case']} / {name}"
    S, A = fr.ref.sums(*up, drop_flagged=False)
    assert torch.isfinite(acc).all(), what
    assert not acc[:, 18:].any(), f"{what}: slots 18-19 not zero"
    dead = ~fr.ref.reached
    assert not acc[dead].any(), f"{what}: Gaussian {int((acc[dead] != 0).any(1).nonzero()[0, 0])} is reached by no " \
                                f"pixel with upstream but has a non-zero sum"
    r, i, c = R.worst_ratio(acc[:, :18], S, A)
    assert r <= 1, f"{what}: Gaussian {i} {R.NAMES[c]}: gpu {float(acc[i, c]):.9g} ref {float(S[i, c]):.9g} at " \
                   f"{r:.3g} x the bound ({float(R.EPS * A[i, c]):.3g})"
    none = lambda *groups: not acc[:, sum((SLOTS[g] for g in groups), [])].any()
    if name == "image":
        assert none("normal"), what
    if name == "normal":
        assert none("rgb"), what
    if name in ("D", "1-T", "distortion"):
        assert none("normal", "rgb"), what
    if name == "median":
        assert none("rgb", "normal", "opacity"), what
        med_w, med_id = fr.allmap[7].reshape(-1), fr.allmap[8].reshape(-1).long()
        keep = (med_w > 0) & (up[1][5].reshape(-1) != 0)  # `up` is masked: ambiguous pixels carry none
        want = torch.zeros(fr.P, dtype=torch.bool)
        want[med_id[keep]] = True
        assert torch.equal((acc[:, :18] != 0).any(1), want), f"{what}: median gradient not on the forward's median ids"
    if name == "channels 7-8":
        assert not acc.any(), what
    return r, S, A


def check_forward(fr):
    """Per-pixel forward maps against the reference's walk on unflagged pixels -> worst error / bound."""
    mp, ref64 = fr.ref.maps(), fr.ref
    ok = ref64.built & ~ref64.flag
    okm = ok & ~ref64.flag_median
    HW = fr.W * fr.H
    img, am = fr.color.reshape(3, HW), fr.allmap.reshape(9, HW)
    worst = 0.0
    for key, got, mask in (("image", img, ok), ("D", am[0], ok), ("1-T", am[1], ok), ("normal", am[2:5], ok),
                           ("median depth", am[5], okm), ("distortion", am[6], ok)):
        v, a = mp[key]
        r, i, _ = R.worst_ratio(got[..., mask].reshape(-1), v[..., mask].reshape(-1), a[..., mask].reshape(-1))
        assert r <= 1, f"{fr.s['case']}: forward {key} at {r:.3g} x the bound"
        worst = max(worst, r)
    mid = torch.where(am[7] > 0, am[8].long(), torch.full_like(am[8].long(), -1))
    assert torch.equal(mid[okm], mp["median id"][okm]), f"{fr.s['case']}: median id"
    assert torch.equal(am[1][~ref64.covered & ref64.built], torch.zeros(int((~ref64.covered & ref64.built).sum()),
                                                                        dtype=torch.float64))
    return worst


# ---- the projection backward on its own ------------------------------------------------------------------------------
def check_projection(fr, acc, grads):
    """The GPU's accumulator, float64, through autograd of surfel_ref64.project + sh_colors; -> worst error / bound.

    Error model: k_surfel_project_bwd recomputes the per-Gaussian geometry in float32 and applies the transposed chain
    (matrix-vector products of 3-4 terms, the quaternion formulas, the SH basis).  Each Jacobian row d f_k / d x is
    then off by a few tens of u relative to its norm over the input tensor (the rotation-invariant error of small
    matrix products), except the mean2D rows, whose 1 / d with d = Tw'Q Tw carries the condition number
    kappa_d = (9 Tw.x^2 + 9 Tw.y^2 + Tw.z^2) / |d|.  So A_P = sum_k |acc_k| gamma_k |d f_k / d x|_tensor with gamma_k =
    kappa_d for the mean2D rows and 1 otherwise, and EPS_P = 16 u.  The scale and rotation gradients are contractions
    of the world-space gradient of the tangent axes and of the rotation matrix (gs = dL/dt_u . R[:,0] mod, gq = sums of
    q dL/dR), whose rounding is relative to those intermediate vectors: there |d f_k / d x| is replaced by
    |d f_k / d R[:,0]| / s_u (and v) and 2 |q| |d f_k / d R|.  The means2D statistic adds |acc_Tu| . Twbar (and Tv),
    Twbar the magnitude of the sums that form Tw."""
    s = fr.s
    t = ref.scene_tensors(s, "cpu")
    leaves = {k: t[k].requires_grad_(True) for k in ("means3D", "scales", "rotations", "shs", "colors_precomp")
              if t[k] is not None}
    delta = torch.zeros(fr.P, 2, dtype=torch.float64, requires_grad=True)
    leaves["delta"] = delta
    g = ref.project(t["means3D"], t["scales"], t["rotations"], t["viewmatrix"], t["projmatrix"], s["W"], s["H"],
                    s["scale_modifier"], delta)
    Rm = g["R"]  # the rotation matrix, to differentiate with respect to it
    sc = t["scales"].detach() * s["scale_modifier"]
    qn = t["rotations"].detach().norm(dim=1)
    rgb = t["colors_precomp"] if t["colors_precomp"] is not None else ref.sh_colors(t["shs"], s["D"], t["means3D"],
                                                                                    t["campos"])
    F = torch.cat([g["mx"][:, None], g["my"][:, None], g["Tu"], g["Tv"], g["Tw"], g["nv"]], 1)
    live = fr.radii.cpu() > 0
    a = acc[:, :18]
    ks = [k for k in leaves if k != "colors_precomp"]
    ref_g = {k: torch.zeros_like(v) for k, v in leaves.items()}
    mag = {k: torch.zeros_like(v) for k, v in leaves.items()}
    Tw = g["Tw"].detach()
    kd = (9 * Tw[:, 0] ** 2 + 9 * Tw[:, 1] ** 2 + Tw[:, 2] ** 2) / g["d"].detach().abs().clamp(min=1e-300)
    for c in list(range(14)) + [15, 16, 17]:
        fk = F[:, c] if c < 14 else rgb[:, c - 15]
        if not fk.requires_grad:
            continue
        js = torch.autograd.grad(fk.sum(), [leaves[k] for k in ks] + [Rm], retain_graph=True, allow_unused=True)
        gam = kd if c < 2 else torch.ones_like(kd)
        jR = js[-1] if js[-1] is not None else torch.zeros_like(Rm)
        for k, j in zip(ks, js[:-1]):
            if j is None:
                continue
            sh = (-1,) + (1,) * (j.dim() - 1)
            ref_g[k] += a[:, c].reshape(sh) * j
            if k == "scales":  # gs = (dL/dt . R column) mod: rounding relative to |dL/dt| = |dL/dR column| / s
                jn = torch.stack([jR[:, :, 0].norm(dim=1) / sc[:, 0] * s["scale_modifier"],
                                  jR[:, :, 1].norm(dim=1) / sc[:, 1] * s["scale_modifier"]], 1)
            elif k == "rotations":  # gq: sums of q times dL/dR, 2 |q| |dL/dR| per element
                jn = (2 * qn * jR.reshape(fr.P, 9).norm(dim=1))[:, None].expand(fr.P, 4)
            else:
                jn = j.reshape(fr.P, -1).norm(dim=1).reshape(sh)
            mag[k] += (a[:, c].abs() * gam).reshape(sh) * jn
    # the statistic dots the Tu / Tv gradients with Tw recomputed in float32, whose tangent entries cancel for splats
    # facing the camera: their rounding is relative to the magnitude of the sums that form them
    P4 = t["projmatrix"].abs()
    Twb = torch.stack([(Rm[:, :, 0].detach().abs() * sc[:, 0:1]) @ P4[:3, 3], (Rm[:, :, 1].detach().abs() * sc[:, 1:2]) @
                       P4[:3, 3], t["means3D"].detach().abs() @ P4[:3, 3] + P4[3, 3]], 1)
    mag["delta"] = mag["delta"] + torch.stack([(a[:, 2:5].abs() * Twb).sum(1), (a[:, 5:8].abs() * Twb).sum(1)], 1)
    what = fr.s["case"]
    pairs = [("means3D", "means3D"), ("scales", "scales"), ("rotations", "rotations")]
    if "shs" in leaves:
        pairs.append(("shs", "shs"))
    worst = 0.0
    for gk, rk in pairs:
        got, want, A = grads[gk].reshape(fr.P, -1), ref_g[rk].reshape(fr.P, -1), mag[rk].reshape(fr.P, -1)
        r, i, c = R.worst_ratio(got[live], want[live], A[live], eps=EPS_P)
        assert r <= 1, f"{what}: projection backward {gk}, Gaussian {int(live.nonzero()[i])} element {c}: gpu " \
                       f"{float(got[live][i, c]):.9g} ref {float(want[live][i, c]):.9g} at {r:.3g} x the bound"
        worst = max(worst, r)
        assert not got[~live].any(), f"{what}: {gk} of a culled Gaussian"
    m2 = grads["means2D"]
    dd = torch.stack([ref_g["delta"][:, 0] * s["W"] / 2, ref_g["delta"][:, 1] * s["H"] / 2], 1)
    dA = torch.stack([mag["delta"][:, 0] * s["W"] / 2, mag["delta"][:, 1] * s["H"] / 2], 1)
    r, i, c = R.worst_ratio(m2[live, :2], dd[live], dA[live], eps=EPS_P)
    assert r <= 1, f"{what}: means2D statistic of Gaussian {int(live.nonzero()[i])}, component {c}, at {r:.3g} x the bound"
    worst = max(worst, r)
    assert not m2[:, 2].any() and not m2[~live].any()
    # straight copies of the accumulator
    assert torch.equal(grads["opacity"].reshape(-1)[live], a[live, 14].float().double())
    assert torch.equal(grads["colors"][live], a[live, 15:18].float().double())
    # exact zeros: culled Gaussians, live Gaussians with an all-zero accumulator, SH rows past the degree
    zero_acc = live & ~(a != 0).any(1)
    for k, v in grads.items():
        assert not v[~live].any(), (what, k)
        assert not v[zero_acc].any(), (what, k)
    if "shs" in leaves:
        assert not grads["shs"][:, (s["D"] + 1) ** 2:].any(), what
        # a clamped colour channel passes no SH gradient (its dL_dcolors keeps the value)
        cl = torch.stack([(fr.clamped.long() >> c) & 1 for c in range(3)], 1).bool() & live[:, None]
        assert not grads["shs"][:, :, :].permute(0, 2, 1)[cl].any(), what
    return worst


# ---- scenes -----------------------------------------------------------------------------------------------------------
SCENES = {
    "random": lambda: ss.scene("random", D=1),
    "sphere": lambda: ss.scene("sphere", colors=True, W=183, H=135),
    "grazing": lambda: ss.scene("grazing", D=0),
    "near": lambda: ss.scene("near", D=2),
    "stacks": lambda: ss.scene("stacks", D=3, bg=(0.3, 0.5, 1.0)),
    "plane": lambda: ss.scene("plane", D=0),
    "modifier": lambda: ss.scene("random", D=3, scale_modifier=0.8, W=40, H=37, seed=5),
    "deep": lambda: view_scene("deep", 40, 36, 1),
    "saturating": lambda: view_scene("saturating", 64, 48, 2),
    "thin": lambda: view_scene("thin", 64, 48, 3, D=1),
    "partial13x7": lambda: view_scene("partial", 13, 7, 4),
    "partial250x170": lambda: view_scene("partial", 250, 170, 5, D=2),
    "offscreen_large": lambda: view_scene("offscreen_large", 160, 120, 6),
}


def scene_properties(key, fr):
    """What each scene is there for, asserted on the GPU's own records."""
    r = fr.ref
    if key == "deep":
        t = max(r.tiles, key=lambda tl: tl["ids"].numel())
        last = r.last[t["pid"]]
        assert t["ids"].numel() > 512, t["ids"].numel()
        assert int(last.max()) % 256 != 0 and int(last.max()) > 256, int(last.max())
        assert float(r.maps()["final T"][t["pid"]].min()) > 1e-4
        # the backward stages its batches from the top of the tile's walk (s_maxc) down: the 256-record batch that
        # holds a pixel's last contributor is (s_maxc - last) // 256
        smax = int(last.max())
        assert len(set(((smax - last[last > 0]) // 256).tolist())) > 1
    if key == "saturating":
        assert r.clamped_pairs >= 20, r.clamped_pairs
        mixed = 0
        for tl in r.tiles:
            e = r.ended[tl["pid"]]
            mixed += int(len(set(r.last[tl["pid"]][e].tolist())) > 1)
        assert mixed >= 2, mixed
    if key == "thin":
        live = fr.radii.cpu() > 0
        d = fr.rec["depth"][live]
        assert len(d) - len(torch.unique(d)) >= 20
    if key.startswith("partial"):
        cov = r.covered.reshape(fr.H, fr.W)
        assert cov[-1].any() and cov[:, -1].any() and fr.W % 16 and fr.H % 16
    if key == "offscreen_large":
        m2 = fr.rec["mean2D"].double()
        off = (m2[:, 0] < 0) | (m2[:, 0] >= fr.W) | (m2[:, 1] < 0) | (m2[:, 1] >= fr.H)
        rc, _, _ = R.surfel_rects(fr.rec["mean2D"], fr.radii.cpu(), fr.W, fr.H)
        area = torch.as_tensor((rc[:, 2] - rc[:, 0]) * (rc[:, 3] - rc[:, 1]))
        S, _ = r.sums(*patterns(fr.W, fr.H, 0)["random"])
        reached = (S != 0).any(1)
        assert int((off & (area > 32) & reached).sum()) >= 5, int((off & (area > 32) & reached).sum())
        sc = torch.as_tensor(fr.s["scales"])
        needle = (sc.max(1).values / sc.min(1).values) >= 99
        assert int((needle & reached).sum()) >= 20
    if key == "modifier":
        t = ref.scene_tensors(fr.s, "cpu")
        g = ref.project(t["means3D"], t["scales"], t["rotations"], t["viewmatrix"], t["projmatrix"], fr.W, fr.H)
        nr = ref.rotmat(t["rotations"])[:, :, 2] @ t["viewmatrix"][:3, :3]
        facing = (nr * g["pv"]).sum(1)
        live = fr.radii.cpu() > 0
        assert (facing[live] > 0).any() and (facing[live] < 0).any()  # both normal flips
        assert fr.clamped[live].any()                                   # clamped SH colour channels


def run_scene(key, fr=None, region=None, names=None, projection=True):
    fr = fr or Frame(SCENES[key]())
    st = fr.ref.stats()
    budget = MAX_FLAGGED_GRAZING if key == "grazing" else MAX_FLAGGED
    print(f"\n{key}: {st}")
    assert st["frac"] < budget, (key, st)
    scene_properties(key, fr)
    fw = check_forward(fr)
    worst, worst_p, dist_err = 0.0, 0.0, None
    for name, up in patterns(fr.W, fr.H, sum(map(ord, key)), region).items():
        if names is not None and name not in names:
            continue
        up = fr.ref.masked(*up)
        acc, grads = fr.backward(*up)
        r, S, A = check_backward(fr, name, up, acc)
        worst = max(worst, r)
        if name == "channels 7-8":
            assert all(not v.any() for v in grads.values()), key
        if name == "distortion":
            dist_err = float((acc[:, :18] - S).abs().sum() / S.abs().sum().clamp(min=1e-300))
        if projection and name in ("random", "image", "median", "pixel last"):
            worst_p = max(worst_p, check_projection(fr, acc, grads))
    print(f"\n{key}: compositing backward worst error / bound {worst:.3g}, forward {fw:.3g}, projection backward "
          f"{worst_p:.3g}; of {st['covered']} covered pixels {100 * st['frac']:.2f} % flagged, "
          f"{100 * st['median_frac']:.2f} % with an ambiguous median; distortion-only relative error "
          f"{dist_err if dist_err is None else f'{dist_err:.3g}'}; flags {st['kinds']}")
    return fr, worst


@pytest.mark.parametrize("key", list(SCENES))
def test_surfel_backward_and_forward_match_f64_reference(key):
    """Grazing: thin slivers whose rays nearly lie in the splat plane make s = p.xy / p.z ill-conditioned (kappa in
    the hundreds), so the rho3 vs rho2 and z vs 0.2 decisions are ambiguous on a wider band: the budget there is 5 %."""
    run_scene(key)


def test_1080p_sampled_tiles():
    """100k surfels at 1920x1080; the reference is built on the busiest tile, a random pair and the last (partial)
    tile, and every upstream is confined to them."""
    s = ss.scene("random", W=1920, H=1080, P=100000, s0=0.01, D=0)
    s["case"] = "1080p"
    from gaustudio_b200 import _C
    W, H = 1920, 1080
    gx, gy = (W + 15) // 16, (H + 15) // 16
    # the busiest tile by the forward's own alpha map
    f = lambda k: torch.tensor(np.asarray(s[k], dtype=np.float32), device=DEV)
    _, _, radii, allmap, *_ = _C.rasterize_surfels(f("bg"), f("means3D"), torch.empty(0, device=DEV), f("opacities"),
                                                   f("scales"), f("rotations"), 1.0, f("viewmatrix"), f("projmatrix"),
                                                   s["tanfovx"], s["tanfovy"], H, W, f("shs"), 0, f("campos"), False,
                                                   False)
    alpha_t = torch.nn.functional.avg_pool2d(allmap[1:2, :1072], 16).flatten().cpu()
    busy = int(alpha_t.argmax())
    ty, tx = divmod(busy, gx)
    rng = np.random.RandomState(4)
    tiles = {ty * gx + tx, int(rng.randint(gx * gy)), int(rng.randint(gx * gy)), gx * gy - 1}
    region = torch.zeros(H, W)
    for t in tiles:
        y, x = divmod(t, gx)
        region[y * 16:(y + 1) * 16, x * 16:(x + 1) * 16] = 1
    fr = Frame(s, tiles=tiles)
    assert int((fr.radii > 0).sum()) > 90000
    run_scene("1080p", fr=fr, region=region, names=("random", "image", "distortion", "median", "spread"),
              projection=False)
