"""-m gpu: the exact tile culling at its edges, on the device's own records, against the float64 checks of
tests/cull_ref64.py.

Scenes are the edge families of cull_ref64 (needles at the dilation's condition-number limit, huge Gaussians centred
5000 px off-screen, centres on tile and pixel boundaries, partial last tiles, opacities at the 0.0039 cut and at
1/255 +- ulps, rects of 32 and 33 tiles, degenerate and indefinite covariances), placed in view space from the wanted
pixel position, depth and screen-space covariance.  Each runs on the un-fused path (SH and colors_precomp), the fused
path (logits, unnormalised rotations), with cov3D_precomp, and on the Mip projection at kernel_size 0, 0.1 and 0.3.
For each scene, once:

  mask         coverage, shape and tightness of every Gaussian's tile mask (cull_ref64.check_mask);
  binning      tile ranges and sorted list equal to test_gpu_binning.reference_binning on the same buffer;
  forward      colour, depth, opacity = 1 - final_T, final_T and the median Gaussian against comp_ref64.Compositing built
               from its own rect lists (nothing culled): test_gpu_first_forward.check_compositing without n_contrib,
               which counts list positions;
  backward     the compositing accumulator against comp_ref64's ten sums (test_gpu_compositing_f64.check), no outlier
               budget;
  reference    on the un-fused paths (SH, colors_precomp, cov3D_precomp; the reference has no Mip and no fused
               activations): colour, depth, median, opacity and radii bit-exact against what the compiled reference
               computed, and the sorted list equal to the reference's list minus provably inert pairs
               (gpu_util.assert_binned_list_is_culled_reference_list): every tile of the small images, the crowded
               tiles and 256 others of the large ones.  Golden data tests/golden/refgold_cull_<family>_<path>.npz
               (tests/refgold.py has the recipe).

On the 8192x4608 images the float64 compositing runs on the four 256x256 corner windows, where the strips and the
partial-tile Gaussians end (the upstream of the backward is zero elsewhere): a dozen float64 planes of the whole image
would not be small."""
import math

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from types import SimpleNamespace

import comp_ref64 as R64
import cull_ref64 as K
import gpu_util as U
import refgold
import scenes
import test_gpu_compositing_f64 as F
import test_gpu_first_forward as FF
from test_gpu_binning import geom_fields, reference_binning

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
PATHS = ("sh", "colors", "fused", "cov3D", "mip0", "mip0.1", "mip0.3")
IMAGES = {"needles": ("250x170", "1920x1080"), "strips": ("17x9", "250x170", "8192x4608"),
          "boundaries": ("17x9", "250x170", "1920x1080"), "partial": ("1x1", "17x9", "250x170", "8192x4608"),
          "opacity": ("250x170", "1920x1080"), "rect32": ("250x170", "1920x1080"), "degenerate": ("17x9", "250x170")}
N_GAUSS = 400
REF_PATHS = ("sh", "colors", "cov3D")
WINDOW = 256  # side of the corner windows of the float64 compositing on the images larger than 1920x1080


def _kernel(path):
    return float(path[3:]) if path.startswith("mip") else None


def lift(f, W, H, path, seed):
    """The screen-space family `f` as 3D Gaussians in the format of scenes.scene: view-space centres from the pixel
    positions at depths 1.5 .. 4, and 3D covariances whose projection J R Sigma R^T J^T (J at the laterally clamped
    centre, as the projection computes it) is the wanted covariance.  Paths with scales and rotations get the nearest
    positive semidefinite covariance."""
    rng = np.random.RandomState(seed)
    cam = scenes.camera(W, H, 50.0)
    tx, ty = math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5)
    fx, fy = W / (2 * tx), H / (2 * ty)
    n = len(f["px"])
    z = rng.uniform(1.5, 4.0, n)
    u, v = ((2 * f["px"] + 1) / W - 1) * tx, ((2 * f["py"] + 1) / H - 1) * ty
    uc, vc = np.clip(u, -1.3 * tx, 1.3 * tx), np.clip(v, -1.3 * ty, 1.3 * ty)
    J = np.zeros((n, 2, 3))
    J[:, 0, 0], J[:, 0, 2] = fx / z, -fx * uc / z
    J[:, 1, 1], J[:, 1, 2] = fy / z, -fy * vc / z
    a, b, c = f["cov"]
    Kc = np.stack([np.stack([a, b], -1), np.stack([b, c], -1)], -2)
    if path != "cov3D":
        w, V = np.linalg.eigh(Kc)
        Kc = V @ (np.maximum(w, 0)[..., None] * np.swapaxes(V, 1, 2))
    Jp = np.swapaxes(J, 1, 2) @ np.linalg.inv(J @ np.swapaxes(J, 1, 2))
    nul = np.cross(J[:, 0], J[:, 1])
    nul /= np.linalg.norm(nul, axis=1, keepdims=True)
    Sv = Jp @ Kc @ np.swapaxes(Jp, 1, 2) + (0.01 * z)[:, None, None] ** 2 * nul[:, :, None] * nul[:, None, :]
    Vm = cam.world_view_transform.double().numpy()
    Rm = Vm[:3, :3]
    Sw = Rm @ Sv @ Rm.T
    means = F._view_to_world(cam, np.stack([u * z, v * z, z], 1))
    o = np.asarray(f["o"], np.float64)
    k = _kernel(path)
    if k is not None:  # the wanted opacity is the filtered one
        o = K.mip_input_opacity(f["cov"], o, k)
    f32 = lambda x: np.ascontiguousarray(x, dtype=np.float32)
    s = dict(case=path, W=W, H=H, D=0, scale_modifier=1.0, bg=np.zeros(3, np.float32), means3D=f32(means),
             opacities=f32(o[:, None]), viewmatrix=cam.world_view_transform.numpy(),
             projmatrix=cam.full_proj_transform.numpy(), campos=cam.camera_center.numpy(), tanfovx=tx, tanfovy=ty)
    if path == "cov3D":
        s["cov3D_precomp"] = f32(np.stack([Sw[:, 0, 0], Sw[:, 0, 1], Sw[:, 0, 2], Sw[:, 1, 1], Sw[:, 1, 2], Sw[:, 2, 2]], 1))
        s["colors_precomp"] = f32(rng.rand(n, 3))
        return s
    w, Q = np.linalg.eigh(Sw)
    Q[:, :, 0] *= np.sign(np.linalg.det(Q))[:, None]
    q = Rotation.from_matrix(Q).as_quat()[:, [3, 0, 1, 2]]
    s["scales"] = f32(np.sqrt(np.maximum(w, 1e-14)))
    s["rotations"] = f32(q)
    if path == "colors":
        s["colors_precomp"] = f32(rng.rand(n, 3))
    else:
        s["shs"] = f32(rng.randn(n, 1, 3))
    if path == "fused":
        s["rotations"] = f32(q * rng.uniform(0.5, 2.0, (n, 1)))
    return s


def args_of(s):
    """The positional arguments of _C.rasterize_gaussians (and of the reference's) for scene `s`, on the device."""
    e = torch.Tensor([])
    d = lambda key: torch.as_tensor(s[key]).to(DEV).contiguous() if s.get(key) is not None else e
    t = {key: d(key) for key in ("means3D", "colors_precomp", "opacities", "scales", "rotations", "cov3D_precomp",
                                 "shs")}
    cam = tuple(torch.as_tensor(np.asarray(s[key], np.float32)).to(DEV).contiguous()
                for key in ("viewmatrix", "projmatrix", "campos"))
    args = (torch.zeros(3, device=DEV), t["means3D"], t["colors_precomp"], t["opacities"], t["scales"],
            t["rotations"], 1.0, t["cov3D_precomp"], cam[0], cam[1], s["tanfovx"], s["tanfovy"], s["H"], s["W"],
            t["shs"], s["D"], cam[2], False, False)
    return t, cam, args


class Scene:
    """One forward of `s` on `path`, its buffers, and backward on given upstream images."""

    def __init__(self, s, path):
        from gaustudio_b200 import _C
        self.s, self.path, self.W, self.H = s, path, s["W"], s["H"]
        self.t, self.cam, args = args_of(s)
        t = self.t
        self.bg = args[0]
        if path == "fused":
            P = t["means3D"].shape[0]
            self.logit = torch.logit(t["opacities"].double()).float().contiguous()
            self.log_scale = torch.log(t["scales"]).contiguous()
            self.f_dc, self.f_rest = t["shs"].contiguous(), torch.zeros(P, 0, 3, device=DEV)
            args = args[:3] + (self.logit, self.log_scale) + args[5:]
            out = _C.rasterize_gaussians(*args, _fused=(self.f_dc, self.f_rest))
        elif _kernel(path) is not None:
            out = _C.rasterize_gaussians_mip(*args, _kernel(path))
        else:
            out = _C.rasterize_gaussians(*args)
        self.out = out
        self.R, color, depth, median, opac, self.radii, self.gb, self.bb, self.ib = out
        self.planes = torch.cat([color, depth, median, opac]).cpu()
        self.P = self.radii.numel()
        ex = _C.debug_export(self.P, self.W, self.H, self.R, self.gb, self.bb, self.ib)
        torch.cuda.synchronize()
        self.ex = {key: (v.cpu() if torch.is_tensor(v) else v) for key, v in ex.items()}

    def backward(self, up):
        from gaustudio_b200 import _C
        s, t, H, W = self.s, self.t, self.H, self.W
        dm = torch.zeros(3, H, W)
        dm[0] = up[2]
        gpu = [up[0].float().to(DEV), up[1].float().reshape(1, H, W).to(DEV), dm.to(DEV),
               up[3].float().reshape(1, H, W).to(DEV)]
        common = (s["tanfovx"], s["tanfovy"], *gpu)
        if self.path == "fused":
            _C.rasterize_gaussians_fused_backward(self.bg, t["means3D"], self.radii, self.f_dc, self.f_rest, self.logit,
                                                  self.log_scale, t["rotations"], 1.0, self.cam[0], self.cam[1],
                                                  *common, s["D"], self.cam[2], self.gb, self.R, self.bb, self.ib, False)
        else:
            args = (self.bg, t["means3D"], self.radii, t["colors_precomp"])
            rest = (t["scales"], t["rotations"], 1.0, t["cov3D_precomp"], self.cam[0], self.cam[1], *common, t["shs"],
                    s["D"], self.cam[2], self.gb, self.R, self.bb, self.ib, False)
            if _kernel(self.path) is not None:
                _C.rasterize_gaussians_mip_backward(*args, t["opacities"], *rest, _kernel(self.path))
            else:
                _C.rasterize_gaussians_backward(*args, *rest)
        acc = _C.debug_accumulator(self.P, self.gb)
        torch.cuda.synchronize()
        return acc.cpu()


def windows(W, H):
    """(x0, y0, w, h) of the pixel windows the float64 compositing covers, tile-aligned."""
    if W * H <= 1920 * 1080:
        return [(0, 0, W, H)]
    return [(x, y, WINDOW, WINDOW) for y in (0, H - WINDOW) for x in (0, W - WINDOW)]


def check_compositing(sc, seed):
    """Forward planes and backward accumulator against the unculled float64 compositing, window by window; the
    backward's upstream is random inside the windows (ambiguous pixels zeroed) and zero outside."""
    W, H = sc.W, sc.H
    ex = sc.ex
    rgb = sc.s["colors_precomp"] if sc.s.get("colors_precomp") is not None else ex["rgb"]
    wins = windows(W, H)
    full = None
    if len(wins) > 1:  # the rect lists of the whole image, cut to each window below
        full, gx, _ = R64.tile_lists(ex["means2D"], sc.radii.cpu(), ex["depths"], W, H)
    g = torch.Generator().manual_seed(seed)
    up = (torch.zeros(3, H, W), torch.zeros(H, W), torch.zeros(H, W), torch.zeros(H, W))
    S = A = 0
    reached = torch.zeros(sc.P, dtype=torch.bool)
    final_T = ex["final_T"].reshape(H, W)
    for x0, y0, w, h in wins:
        m2 = ex["means2D"].double() - torch.tensor([x0, y0], dtype=torch.float64)
        lists = None
        if full is not None:
            lists = [full[(y0 // 16 + ty) * gx + x0 // 16 + tx] for ty in range((h + 15) // 16)
                     for tx in range((w + 15) // 16)]
        comp = R64.Compositing(m2, ex["conic_opacity"], rgb, ex["depths"], sc.radii.cpu(), w, h, np.zeros(3),
                               lists=lists)
        Z = dict(W=w, H=h, r1_planes=sc.planes[:, y0:y0 + h, x0:x0 + w], r1_final_T=final_T[y0:y0 + h, x0:x0 + w])
        FF.check_compositing(Z, comp=comp, n_contrib=False)
        rn = lambda *shape: torch.randn(*shape, generator=g)
        u = comp.masked(rn(3, h, w), rn(h, w), rn(h, w), rn(h, w))
        s_, a_ = comp.sums(*u)
        S, A = S + s_, A + a_
        reached |= comp.reached
        for full_img, part in zip(up, u):
            full_img[..., y0:y0 + h, x0:x0 + w] = part
    acc = sc.backward(up)
    fr = SimpleNamespace(s=sc.s, ref=SimpleNamespace(reached=reached))
    F.check(fr, "random", up, acc, (S, A))


def reference_run(s, img):
    """What the compiled reference returns for scene `s`: the five outputs, and segments of its sorted list (every
    tile of an image of <= 4096 tiles, else the 8 most crowded and 256 other non-empty tiles)."""
    from oracle import ref_driver
    W, H = s["W"], s["H"]
    T = ((W + 15) // 16) * ((H + 15) // 16)
    r = ref_driver.module().rasterize_gaussians(*args_of(s)[2])
    out = {f"{img}_num_rendered": r[0], **{f"{img}_out{i}": r[i] for i in range(1, 6)}}
    rg = ref_driver.parse_image_ranges(r[8], W * H, T)
    pl = ref_driver.parse_binning(r[7], r[0])
    if T <= 4096:
        seg = U.reference_tile_segments(pl, rg, T, T, 0, 0)
    else:
        busy = int(((rg[:T, 1] - rg[:T, 0]) > 0).sum())
        seg = U.reference_tile_segments(pl, rg, T, 8, min(256, max(busy - 8, 0)), 0)
    out.update({f"{k}_{img}": v for k, v in seg.items()})
    return out


def check_reference(sc, ref, img):
    W, H, P = sc.W, sc.H, sc.P
    assert sc.out[0] == ref.scalar(f"{img}_num_rendered"), "num_rendered"
    for i, name in enumerate(("colour", "depth", "median", "opacity", "radii"), 1):
        ref.assert_equal(f"{img}_out{i}", sc.out[i], what=f"{img}: {name}")
    tiles = ref.array(f"seg_tiles_{img}")
    U.assert_binned_list_is_culled_reference_list(sc.ex, ref.array(f"seg_list_{img}"), ref.array(f"seg_ranges_{img}"),
                                                  W, H, P, tiles=tiles)


def run_one(fam, img, path, s, ref):
    W, H = s["W"], s["H"]
    sc = Scene(s, path)
    P = sc.P
    rect, mask, depth, _, splat = geom_fields(sc.gb, P, with_splat=True)
    sp = splat.cpu().numpy()
    rc = rect.cpu().numpy()
    r = dict(px=sp[:, 0], py=sp[:, 1], A=sp[:, 2], B=sp[:, 3], C=sp[:, 4], o=sp[:, 5], tau=sp[:, 11],
             x0=rc[:, 0] & 0xffff, x1=rc[:, 0] >> 16, y0=rc[:, 1] & 0xffff, y1=rc[:, 1] >> 16, W=W, H=H)
    vis = sc.radii.cpu().numpy() > 0
    for key in ("x0", "x1", "y0", "y1"):
        r[key] = np.where(vis, r[key], 0)
    # the records the checks read are the ones the rest of the library sees
    assert torch.equal(torch.as_tensor(sp[vis, :2]), sc.ex["means2D"][torch.as_tensor(vis)])
    rep = K.check_mask(r, mask.cpu().numpy())
    assert not rep.failed(), f"{fam} {img} {path}: {rep.text()}"
    ranges, pl = reference_binning(rect, mask, depth, W, H)
    assert torch.equal(sc.ex["ranges"].long(), ranges.cpu()), "tile ranges differ"
    assert torch.equal(sc.ex["point_list"].long(), pl.cpu()), "point list differs"
    check_compositing(sc, seed=sum(map(ord, fam + img + path)))
    if ref is not None:
        check_reference(sc, ref, img)
    st = dict(rep.stats)
    # on the Mip path a covariance with det0 or det1 <= 1e-6 gets coef 0: opacity exactly 0, an empty mask
    st["zero_o"] = int((vis & (r["o"] == 0)).sum())
    return st


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("fam", K.FAMILIES)
def test_culling_edges(fam, path):
    if fam == "degenerate" and path not in ("cov3D", "mip0"):
        pytest.skip("scales and rotations cannot express an indefinite covariance")
    k = _kernel(path)
    built = []
    for j, img in enumerate(IMAGES[fam]):
        W, H = K.IMAGES[img]
        seed = 1000 * K.FAMILIES.index(fam) + PATHS.index(path) * 10 + j
        f = K.family(fam, N_GAUSS, W, H, seed=seed, dil=0.3 if k is None else k)
        built.append((img, lift(f, W, H, path, seed)))
    ref = None
    if path in REF_PATHS:
        ref = refgold.reference(f"cull_{fam}_{path}",
                                lambda: {key: v for img, s in built for key, v in reference_run(s, img).items()})
    rows = [run_one(fam, img, path, s, ref) for img, s in built]
    tot = lambda key: sum(s[key] for s in rows)
    share = sum(s["tight_share"] * s["set"] for s in rows) / max(tot("set"), 1)
    slack = min(s["slack_min"] for s in rows)
    print(f"\n{fam}/{path}: masked {tot('masked')}, required tiles {tot('required')}, set bits {tot('set')}, "
          f"worst coverage slack {slack:.4f}, tightness share {share:.4f}, worst box/taum "
          f"{max(s['worst_tight'] for s in rows):.4f}, all-ones fallback {tot('fallback')} (flagged {tot('flagged')}), "
          f"o < 0.0039 {tot('dead')} (o = 0: {tot('zero_o')})")
    assert tot("masked") > 0
    if fam == "degenerate" and k is not None:
        # on the Mip path a singular or indefinite cov2D is dead (coef 0) unless float32 rounding leaves det0 above
        # 1e-6, so this scene mostly checks the empty mask of o = 0 and sets too few bits for a tightness share; the
        # all-ones fallback of indefinite conics is the cov3D_precomp scene's
        assert tot("zero_o") >= 0.5 * tot("masked"), (tot("zero_o"), tot("masked"))
        return
    assert share <= (K.MIP0_TIGHT_SHARE if path == "mip0" else K.TIGHT_SHARE)[fam], share
