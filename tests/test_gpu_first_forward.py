"""The first forward of a fresh process, stage by stage (DESIGN.md 3.5's open issue).

`test_fused_path_with_mostly_culled_ctas_matches_unfused` has failed only on the FIRST un-fused forward of its shape in
a process, and only compares final images, so a failure cannot say which stage went wrong.  tests/test_gpu_foreign_state.py
ruled out stale memory, but it renders inputs that were materialised long before.  Here every case runs ONCE in its own
child process (tests/first_forward_child.py): the inputs are produced on the device the way the case prescribes, the
forward is issued at once, its internal state is exported, and the same device tensors are rendered twice more (2: the
speculative form, 3: the plain blocking form the first one took).  The parent judges the child's npz in this order and
names the FIRST stage that fails, with the number of Gaussians / tiles / pixels involved and the largest deviation:

  inputs           what the forward was given equals the CPU float32 evaluation of the same activations: bit for bit for
                   copies and `cat`, within 4 ulp for exp / sigmoid / normalize;
  projection       the per-Gaussian records against the float64 projection (tests/proj_ref64.py, tests/mip_ref64.py) of
                   the downloaded inputs at the bounds of test_gpu_projection_f64.py; radii, tiles touched and clamp bits
                   exact wherever the float64 value pins the decision; and bit-identical to render 3;
  scan             the ranges are one exclusive scan, num_binned is its total, num_rendered the sum of tiles touched;
  scatter+sort     the sorted list is the (own depth bits, index)-ordered rectangle list of the forward's OWN records
                   with only provably inert pairs removed (gpu_util.assert_binned_list_is_culled_reference_list), and,
                   where the CPU oracle's sort keys and tile rectangles are the device's bit for bit, the same against
                   the oracle's list;
  compositing      the 8 planes, n_contrib, final_T and the median Gaussian against the float64 compositing
                   (tests/comp_ref64.py) of the forward's own records and own list, so an upstream error is not counted
                   twice;
  reproducibility  render 1 took the plain path, render 2 was a speculative hit, render 3 plain again; every exported
                   array and plane of render 1 is bit-identical to render 3 (same path) and to render 2 (speculative).

Cases: `materialised` (control: inputs made, device drained, then the forward), `same_stream` (the un-fused
`vanilla_renderer` sequence of the failing test: model.to, cam.to, activations, cat, forward), `same_stream_fused`,
`side_stream_waited` (inputs on a second stream the render stream waits for: INTEGRATION.md's contract),
`non_default_stream` (everything inside `torch.cuda.stream(s)`), `after_allocator_churn` (the forward's torch.empty
blocks recycled from 0xFF-filled blocks freed while their fill kernels are still queued), `eager_modules`
(CUDA_MODULE_LOADING=EAGER), `mip` and `surfel` (the renderers that share the binning; the surfel rasterizer has no
state export, so its stages are inputs and reproducibility of colour, allmap, radii and num_rendered).  Scene: 40 000
Gaussians of cfg 5 from inside at 240x180; `same_stream` also on golden case B and on cfg 1 at 256x256.

Which stream everything runs on (read from gaustudio_b200/_C.py and csrc/gsr_api.cu, exercised by `non_default_stream`
and `side_stream_waited`):
* `_C.rasterize_gaussians*`: `_f32` / `_f32_rot` (`.to(device)`, `.contiguous()`, `.clone()`), `torch.empty` of the
  outputs, `_alloc` of the three scratch buffers and the `pl.rmax` update are torch ops: they run on, and allocate
  for, torch's CURRENT stream, which is the stream handed to the library.  `_bg_on` copies the CPU background once per
  value on the stream current at that first call and caches the device tensor; the forward never reads the background
  (the backward does, on whatever stream it runs: a cached copy made on another stream is ordered only by the blocking
  pageable copy that made it, which has completed on the host before `.to` returned).
* `gsr_api.cu`, forward entry points: `cudaMemsetAsync(tile_count)`, `k_init_header`, projection, scan, the 16-byte count
  copy, `k_set_capacity`, scatter, sort, compositing all take `h.stream`.  No call uses the legacy default stream.  The
  plain path copies the counts into pageable stack memory (the copy returns when done) and then synchronises the
  stream; the speculative path copies into 16 pinned bytes owned by the host thread and reads them only after
  `cudaEventSynchronize` on an event recorded right behind the copy.
* host state: the hint table `g_hints` is read and written under `g_hint_mu`; `SpecHost` (pinned counts + event) is
  `thread_local`, and a forward blocks on its event before it returns, so one thread never has two forwards sharing
  `counts` in flight, whatever streams it alternates between.
* once-per-device `cudaFuncSetAttribute` calls (sort tiers, the projection's staging block) are made on the host right
  before the first launch that needs them, on every path; the flags that remember them are per device.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import comp_ref64 as C64
import gpu_util as U
import mip_ref64 as MR
import proj_ref64 as R
import scenes
from test_proj_ref64 import ATOL, NEAR_LIMIT, RTOL

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CHILD = os.path.join(HERE, "first_forward_child.py")
STAGES = ("inputs", "projection", "scan", "scatter+sort", "compositing", "reproducibility")
RECORDS = ("means2D", "conic_opacity", "depths", "rgb", "cov3D", "clamped", "tiles_touched")
EXPORTS = RECORDS + ("ranges", "point_list", "n_contrib", "final_T")
ULPS = 4  # exp / sigmoid / normalize on the device against the CPU's float32 evaluation


class StageFailure(AssertionError):
    def __init__(self, stage, msg):
        super().__init__(f"first failing stage: {stage}: {msg}")
        self.stage = stage


def _need(stage, ok, msg):
    if not ok:
        raise StageFailure(stage, msg() if callable(msg) else msg)


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def _tiles_of(mask_hw):
    """number of 16x16 tiles with a set pixel, of an [H,W] mask"""
    H, W = mask_hw.shape
    pad = np.zeros(((H + 15) // 16 * 16, (W + 15) // 16 * 16), bool)
    pad[:H, :W] = mask_hw
    return int(pad.reshape(pad.shape[0] // 16, 16, pad.shape[1] // 16, 16).any(axis=(1, 3)).sum())


def _near_int(x, rel=2e-4):
    x = np.asarray(x, np.float64)
    return ~(np.abs(x - np.round(x)) > rel * (1 + np.abs(x)))  # NaN counts as near


# ---- stage: inputs -----------------------------------------------------------------------------------------------------
def check_inputs(Z):
    rounded = [str(k) for k in np.asarray(Z["rounded"]).reshape(-1)]  # the inputs a device activation produced
    for key in sorted(k[4:] for k in Z if k.startswith("exp_")):
        a, b = np.asarray(Z["in_" + key]), np.asarray(Z["exp_" + key])
        _need("inputs", a.size == b.size, f"{key}: the forward was given {a.shape}, expected {b.shape}")
        a = a.reshape(b.shape)
        if key in rounded:
            bad = ~(np.abs(a.astype(np.float64) - b) <= ULPS * np.spacing(np.abs(b)).astype(np.float64))
            dev = np.abs(a.astype(np.float64) - b) / np.spacing(np.abs(b)).astype(np.float64)
            _need("inputs", not bad.any(), lambda: f"{key}: {int(bad.sum())} of {bad.size} elements beyond {ULPS} ulp of "
                  f"the CPU float32 activation (worst {np.nanmax(dev):.3g} ulp, rows {np.unique(np.nonzero(bad)[0])[:5]})")
        else:
            bad = _bits(a) != _bits(b)
            _need("inputs", not bad.any(), lambda: f"{key}: {int(bad.sum())} of {bad.size} elements are not the bits of "
                  f"the CPU tensor (largest deviation {np.nanmax(np.abs(a.astype(np.float64) - b)):.3g})")


# ---- stage: projection -------------------------------------------------------------------------------------------------
def _stored(Z, keys):
    """`keys` without cov3D when the covariance came precomputed: the forward then stores none, and the export of that
    field is whatever the buffer held"""
    pre = np.asarray(Z.get("in_cov3D_precomp", np.zeros(0))).size > 0
    return [k for k in keys if not (pre and k == "cov3D")]


def _params(Z):
    g = lambda k: Z["in_" + k] if "in_" + k in Z and np.asarray(Z["in_" + k]).size else None
    if bool(Z["fused"]):
        return dict(means3D=g("means3D"), f_dc=g("f_dc"), f_rest=g("f_rest"), opacity_logits=g("opacities"),
                    log_scales=g("scales"), raw_rotations=g("rotations"))
    return {k: g(k) for k in R.UNFUSED_KEYS}


def projection_reference(Z):
    """Float64 records of every Gaussian from the inputs the forward was given, and where float32 decisions are pinned."""
    fused, W, H = bool(Z["fused"]), int(Z["W"]), int(Z["H"])
    params = {k: v for k, v in _params(Z).items() if v is not None}
    cam = R.camera(Z["in_viewmatrix"], Z["in_projmatrix"], Z["in_campos"], float(Z["in_tanfovx"]), float(Z["in_tanfovy"]),
                   W, H, int(Z["in_D"]), float(Z["in_scale_modifier"]))
    if str(Z["kind"]) == "mip":
        f = MR.forward(params, cam, float(Z["kernel_size"]))
        ok = ((f["det0"] / MR.EPS6 - 1).abs() > 1e-2) & ((f["det1"] / MR.EPS6 - 1).abs() > 1e-2)
    else:
        with torch.no_grad():
            s = R._state(R._params(params, fused), cam, fused)
        f = dict(R.forward(params, cam, fused), cov2D=s["cov2D"], opacity=s["opacity"], color_raw=s["color_raw"])
        ok = torch.ones(f["depth"].shape[0], dtype=torch.bool)
    a, b, c = f["cov2D"].unbind(1)
    det, mid = a * c - b * b, 0.5 * (a + c)
    sq = torch.sqrt(torch.clamp(mid * mid - det, min=0.1))
    f["pre_ceil"] = 3 * torch.sqrt(torch.maximum(mid + sq, mid - sq))
    ri = f["radius"]  # 0 where the reference culls; the rect of the un-culled radius decides visibility
    rr = torch.nan_to_num(torch.ceil(f["pre_ceil"]), nan=0.0, posinf=0.0)
    px, py = f["means2D"].unbind(1)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    edges = [(px - rr) / 16, (px + rr + 15) / 16, (py - rr) / 16, (py + rr + 15) / 16]
    rect = lambda v, hi: torch.clamp(torch.trunc(v), min=0).clamp(max=hi)
    tiles = (rect(edges[1], gx) - rect(edges[0], gx)) * (rect(edges[3], gy) - rect(edges[2], gy))
    f["tiles"] = torch.where(ri > 0, torch.nan_to_num(tiles), torch.zeros_like(tiles)).to(torch.int64)
    lat = ((f["txtz_over_lim"].abs() - 1).abs() >= NEAR_LIMIT).all(1)
    cond = (det > 1e-3 * a * c) & torch.isfinite(f["pre_ceil"])
    f["pinned"] = (lat & ok & cond).numpy()
    f["sure"] = f["pinned"] & ~_near_int(f["pre_ceil"].numpy()) & (np.abs(f["depth"].numpy() - 0.2) > 1e-5) \
        & ~np.any([_near_int(e.numpy()) for e in edges], axis=0)
    return f


def check_projection(Z, f=None):
    f = projection_reference(Z) if f is None else f
    radii, P = Z["r1_radii"], Z["r1_radii"].shape[0]
    sure, vis = f["sure"], radii > 0
    want = f["radius"].numpy()
    bad = sure & (radii != want)
    _need("projection", not bad.any(), lambda: f"radii: {int(bad.sum())} of {int(sure.sum())} pinned Gaussians differ from "
          f"the float64 radius (largest deviation {int(np.abs(radii - want)[bad].max())}, first #{int(np.nonzero(bad)[0][0])})")
    tt = Z["r1_tiles_touched"].astype(np.int64)
    bad = sure & (tt != f["tiles"].numpy())
    _need("projection", not bad.any(), lambda: f"tiles_touched: {int(bad.sum())} of {int(sure.sum())} pinned Gaussians "
          f"differ (largest deviation {int(np.abs(tt - f['tiles'].numpy())[bad].max())}, first #{int(np.nonzero(bad)[0][0])})")
    m = vis & f["pinned"]
    co = Z["r1_conic_opacity"]
    pairs = [("means2D", Z["r1_means2D"], f["means2D"]), ("conic", co[:, :3], f["conic"]),
             ("opacity", co[:, 3:4], f["opacity"].reshape(-1, 1)), ("depths", Z["r1_depths"], f["depth"])]
    if np.asarray(Z.get("in_colors_precomp", np.zeros(0))).size == 0:
        pairs.append(("rgb", Z["r1_rgb"], f["rgb"]))
    if np.asarray(Z.get("in_cov3D_precomp", np.zeros(0))).size == 0 and str(Z["kind"]) == "3dgs":
        pairs.append(("cov3D", Z["r1_cov3D"], f["cov3D"]))
    for name, a, b in pairs:
        r, i, n = R.row_check(torch.as_tensor(np.asarray(a)), b, RTOL, ATOL, m)
        _need("projection", r <= 1, lambda: f"{name}: {n} of {int(m.sum())} visible Gaussians beyond the float64 bound, "
              f"worst #{i} at {r:.3g} x the bound (gpu {np.asarray(a)[i]}, float64 {b[i].numpy()})")
    if "color_raw" in f and any(p[0] == "rgb" for p in pairs):
        raw = f["color_raw"].numpy()
        known = vis[:, None] & (np.abs(raw) > 1e-5)
        bad = known & (Z["r1_clamped"].astype(bool) != (raw < 0))
        _need("projection", not bad.any(), lambda: f"clamped: {int(bad.any(1).sum())} Gaussians with a wrong clamp bit")
    for k in _stored(Z, RECORDS + ("radii",)):
        a, b = Z["r1_" + k], Z["r3_" + k]
        bad = (_bits(a) != _bits(b)).reshape(P, -1).any(1)
        _need("projection", not bad.any(), lambda: f"{k}: {int(bad.sum())} of {P} Gaussians differ between the first forward "
              f"and the plain-path re-render (largest deviation "
              f"{np.nanmax(np.abs(a.astype(np.float64) - b.astype(np.float64))):.3g}, first #{int(np.nonzero(bad)[0][0])})")


# ---- stage: scan -------------------------------------------------------------------------------------------------------
def check_scan(Z):
    rg = Z["r1_ranges"].astype(np.int64)
    n = rg[:, 1] - rg[:, 0]
    T, nb = rg.shape[0], int(Z["r1_num_binned"])
    _need("scan", (n >= 0).all(), lambda: f"{int((n < 0).sum())} of {T} tiles have a negative range")
    _need("scan", not rg[n == 0].any(), lambda: f"{int(rg[n == 0].any(1).sum())} empty tiles have a non-zero range")
    live = rg[n > 0]
    if len(live):
        _need("scan", live[0, 0] == 0, lambda: f"the first non-empty range starts at {live[0, 0]}, not 0 "
              f"({len(live)} of {T} tiles non-empty)")
        gap = live[1:, 0] != live[:-1, 1]
        _need("scan", not gap.any(), lambda: f"{int(gap.sum())} of {len(live)} non-empty ranges do not start where the "
              f"previous one ends (largest gap {int(np.abs(live[1:, 0] - live[:-1, 1]).max())})")
    total = int(live[-1, 1]) if len(live) else 0
    _need("scan", total == nb, f"the ranges end at {total} but num_binned is {nb}")
    _need("scan", Z["r1_point_list"].shape[0] == nb, f"point_list has {Z['r1_point_list'].shape[0]} entries, num_binned {nb}")
    rect = int(Z["r1_tiles_touched"].astype(np.int64).sum())
    _need("scan", int(Z["r1_R"]) == rect, f"num_rendered {int(Z['r1_R'])} is not the sum of tiles_touched {rect}")


# ---- stage: scatter + sort ---------------------------------------------------------------------------------------------
def _export_tensors(Z):
    """the first forward's export as gpu_util.assert_binned_list_is_culled_reference_list takes it (CPU tensors)"""
    ex = {k: torch.as_tensor(Z["r1_" + k].astype(np.int64)) for k in ("point_list", "ranges")}
    ex.update({k: torch.as_tensor(np.asarray(Z["r1_" + k])) for k in ("means2D", "conic_opacity")})
    ex["num_binned"] = int(Z["r1_num_binned"])
    return ex


def _own_lists(Z):
    """per-tile lists of the forward's own sorted list"""
    pl, rg = Z["r1_point_list"].astype(np.int64), Z["r1_ranges"].astype(np.int64)
    return [pl[a:b].tolist() for a, b in rg]


def _list_check(Z, ref_pl, ref_rg, what):
    W, H, P = int(Z["W"]), int(Z["H"]), Z["r1_radii"].shape[0]
    try:
        return U.assert_binned_list_is_culled_reference_list(_export_tensors(Z), ref_pl, ref_rg, W, H, P)
    except AssertionError as e:
        # which tiles: compare tile by tile as sets / sequences
        pl, rg = Z["r1_point_list"].astype(np.int64), Z["r1_ranges"].astype(np.int64)
        rrg, rpl = np.asarray(ref_rg).astype(np.int64).reshape(-1, 2), np.asarray(ref_pl).astype(np.int64)
        foreign = order = 0
        for t in range(rg.shape[0]):
            ours, ref = pl[rg[t, 0]:rg[t, 1]], rpl[rrg[t, 0]:rrg[t, 1]]
            if not np.isin(ours, ref).all() or len(set(ours.tolist())) != len(ours):
                foreign += 1
            elif not np.array_equal(ref[np.isin(ref, ours)], ours):
                order += 1
        raise StageFailure("scatter+sort", f"{what}: {e}; of {rg.shape[0]} tiles, {foreign} hold an instance that is not "
                           f"theirs (or hold one twice) and {order} more are out of order") from None


def _rects(means2D, radii, W, H):
    """[P,4] tile rectangles (x0, y0, x1, y1) of getRect on float32 means and integer radii"""
    gx, gy = (W + 15) // 16, (H + 15) // 16
    m, r = np.asarray(means2D, np.float32), np.asarray(radii).astype(np.float32)
    lo = lambda v, hi: np.clip(np.trunc((v - r) / np.float32(16)), 0, hi)
    hi_ = lambda v, hi: np.clip(np.trunc((v + r + np.float32(15)) / np.float32(16)), 0, hi)
    return np.stack([lo(m[:, 0], gx), lo(m[:, 1], gy), hi_(m[:, 0], gx), hi_(m[:, 1], gy)], 1).astype(np.int64)


def check_scatter_sort(Z):
    W, H = int(Z["W"]), int(Z["H"])
    lists, gx, gy = C64.tile_lists(Z["r1_means2D"], Z["r1_radii"], Z["r1_depths"], W, H)
    ends = np.cumsum([len(x) for x in lists])
    own_rg = np.stack([ends - [len(x) for x in lists], ends], 1)
    own_pl = np.concatenate([np.asarray(x, np.int64) for x in lists]) if ends[-1] else np.zeros(0, np.int64)
    _list_check(Z, own_pl, own_rg, "against the (depth, index)-sorted rectangle lists of the forward's own records")
    if str(Z["kind"]) != "3dgs" or bool(Z["fused"]):
        return None
    # the pinned CPU oracle on the inputs the forward was given: its list is the reference's
    from oracle.oracle import Oracle
    g = lambda k: Z["in_" + k] if "in_" + k in Z and np.asarray(Z["in_" + k]).size else None
    o = Oracle()
    out = o.forward(g("means3D"), g("opacities"), Z["in_viewmatrix"], Z["in_projmatrix"], Z["in_campos"],
                    float(Z["in_tanfovx"]), float(Z["in_tanfovy"]), W, H, int(Z["in_D"]), shs=g("shs"),
                    colors_precomp=g("colors_precomp"), scales=g("scales"), rotations=g("rotations"),
                    cov3D_precomp=g("cov3D_precomp"), scale_modifier=float(Z["in_scale_modifier"]))
    geo = o.geometry()
    vis = Z["r1_radii"] > 0
    same_keys = np.array_equal(out["radii"], Z["r1_radii"]) and \
        np.array_equal(_bits(geo["depths"])[vis], _bits(Z["r1_depths"])[vis]) and \
        np.array_equal(_rects(geo["means2D"], out["radii"], W, H)[vis], _rects(Z["r1_means2D"], Z["r1_radii"], W, H)[vis])
    # host libm can move a key or a rectangle edge by an ulp: the oracle's list is the device's reference only where its
    # sort keys and tile rectangles are the device's
    if same_keys:
        ob = o.binning()
        _list_check(Z, ob["point_list"], ob["ranges"], "against the CPU oracle's list")
    return same_keys


# ---- stage: compositing ------------------------------------------------------------------------------------------------
def check_compositing(Z, comp=None, n_contrib=True):
    """The planes, final_T, n_contrib and median of Z's render 1 against the float64 compositing of its records.
    comp: the comp_ref64.Compositing to compare with (default: the one of the forward's own sorted list);
    n_contrib=False leaves n_contrib out (it counts list positions, so it is comparable on the forward's own lists
    only).  -> comp.stats()."""
    W, H = int(Z["W"]), int(Z["H"])
    HW = W * H
    if comp is None:
        pre = np.asarray(Z.get("in_colors_precomp", np.zeros(0)))
        rgb = pre if pre.size else Z["r1_rgb"]
        comp = C64.Compositing(Z["r1_means2D"], Z["r1_conic_opacity"], rgb, Z["r1_depths"], Z["r1_radii"], W, H,
                               np.zeros(3), lists=_own_lists(Z))
    ref = torch.zeros(5, HW, dtype=torch.float64)   # r, g, b, depth, and their common magnitude scale below
    mag = torch.zeros(5, HW, dtype=torch.float64)
    kmax = torch.zeros(HW, dtype=torch.float64)
    for tl in comp.tiles:
        ids, pid, w, gain = tl["ids"], tl["pid"], tl["w"], tl["gain"]
        vals = [comp.rgb[ids, j] for j in range(3)] + [comp.depth[ids]]
        for j, v in enumerate(vals):
            ref[j, pid] = (w * v[None, :]).sum(1)
            mag[j, pid] = (w * v[None, :].abs() * gain).sum(1)
        kmax[pid] = gain.max(1).values
    planes = torch.as_tensor(Z["r1_planes"]).double().reshape(8, HW)
    ok = ~comp.flag
    what = ("red", "green", "blue", "depth")
    for j, p in enumerate((0, 1, 2, 3)):
        err = (planes[p] - ref[j]).abs()
        bad = ok & ~(err <= C64.EPS * mag[j] + 1e-7)
        _need("compositing", not bad.any(), lambda: f"{what[j]}: {int(bad.sum())} pixels in "
              f"{_tiles_of(bad.reshape(H, W).numpy())} tiles beyond the float64 bound (largest deviation "
              f"{float(err[bad].max()):.3g}, {float((err / (C64.EPS * mag[j] + 1e-7))[bad].max()):.3g} x the bound)")
    fT = torch.as_tensor(Z["r1_final_T"]).double().reshape(HW)
    err = (fT - comp.final_T).abs()
    bad = ok & ~(err <= C64.EPS * kmax * comp.final_T + 1e-7)
    _need("compositing", not bad.any(), lambda: f"final_T: {int(bad.sum())} pixels in {_tiles_of(bad.reshape(H, W).numpy())} "
          f"tiles beyond the float64 bound (largest deviation {float(err[bad].max()):.3g})")
    bad = ok & (planes[7] != (1 - torch.as_tensor(Z["r1_final_T"]).reshape(HW)).double())
    _need("compositing", not bad.any(), lambda: f"opacity: {int(bad.sum())} pixels are not 1 - final_T")
    if n_contrib:
        nc = torch.as_tensor(Z["r1_n_contrib"].astype(np.int64)).reshape(HW)
        bad = ok & (nc != comp.last)
        _need("compositing", not bad.any(), lambda: f"n_contrib: {int(bad.sum())} pixels in "
              f"{_tiles_of(bad.reshape(H, W).numpy())} tiles differ (largest deviation "
              f"{int((nc - comp.last).abs()[bad].max())})")
    okm = ok & ~comp.flag_median
    has = planes[5] > 0
    bad = okm & (has != (comp.median >= 0))
    _need("compositing", not bad.any(), lambda: f"median: {int(bad.sum())} pixels disagree on whether T crosses 0.5")
    bad = okm & has & (planes[6].long() != comp.median)
    _need("compositing", not bad.any(), lambda: f"median id: {int(bad.sum())} pixels in "
          f"{_tiles_of(bad.reshape(H, W).numpy())} tiles name another Gaussian")
    return comp.stats()


# ---- stage: reproducibility --------------------------------------------------------------------------------------------
def check_reproducibility(Z):
    st = np.asarray(Z["spec_stats"]).astype(np.int64)
    d = np.diff(st, axis=0)  # (hits, redos) of renders 1, 2, 3
    if str(Z["kind"]) != "surfel":  # the surfel forward has no speculative form
        _need("reproducibility", tuple(d[0]) == (0, 0), f"the first forward took the speculative path {tuple(d[0])}")
        _need("reproducibility", d[1].sum() == 1, f"render 2 was not speculative (hits, redos) = {tuple(d[1])}")
        _need("reproducibility", tuple(d[2]) == (0, 0), f"render 3 did not take the plain path {tuple(d[2])}")
    H, W = int(Z["H"]), int(Z["W"])
    keys = [k for k in _stored(Z, EXPORTS + ("planes", "radii", "R", "num_binned")) if "r1_" + k in Z]
    for other, name in ((3, "the plain-path re-render"), (2, "the speculative re-render")):
        for k in keys:
            a, b = np.asarray(Z["r1_" + k]), np.asarray(Z[f"r{other}_{k}"])
            _need("reproducibility", a.shape == b.shape, f"{k}: shape {a.shape} in the first forward, {b.shape} in {name}")
            bad = _bits(a) != _bits(b)
            if not bad.any():
                continue
            dev = np.nanmax(np.abs(a.astype(np.float64) - b.astype(np.float64)))
            if k in ("planes", "n_contrib", "final_T"):
                m = bad.reshape(-1, H, W).any(0)
                where = f"{int(m.sum())} pixels in {_tiles_of(m)} of {((H + 15) // 16) * ((W + 15) // 16)} tiles"
            elif a.ndim == 0:
                where = f"{int(a)} against {int(b)}"
            else:
                where = f"{int(bad.reshape(len(bad), -1).any(1).sum())} of {len(bad)} rows"
            raise StageFailure("reproducibility", f"{k} of the first forward differs from {name}: {where}, largest "
                               f"deviation {dev:.3g}")


def judge(Z):
    """Run the stages in order on a child's npz (a dict of arrays); raises StageFailure at the first one that fails.
    -> dict of notes for the report."""
    notes = {}
    check_inputs(Z)
    if str(Z["kind"]) != "surfel":
        check_projection(Z)
        check_scan(Z)
        notes["oracle_list_compared"] = check_scatter_sort(Z)
        notes["flags"] = check_compositing(Z)
    check_reproducibility(Z)
    return notes


# ---- CPU: the checkers on the oracle's own state, clean and with seeded faults ----------------------------------------
def oracle_npz(case="A"):
    """What a child would write, made from the CPU oracle's state of a small scene (all three renders the same)."""
    from oracle.oracle import Oracle
    s = scenes.scene(case)
    W, H, P = s["W"], s["H"], s["means3D"].shape[0]
    o = Oracle()
    out = o.forward(s["means3D"], s["opacities"], s["viewmatrix"], s["projmatrix"], s["campos"], s["tanfovx"],
                    s["tanfovy"], W, H, s["D"], shs=s.get("shs"), colors_precomp=s.get("colors_precomp"),
                    scales=s.get("scales"), rotations=s.get("rotations"), cov3D_precomp=s.get("cov3D_precomp"),
                    scale_modifier=s["scale_modifier"])
    geo, b = o.geometry(), o.binning()
    Z = dict(case=np.array("oracle"), scene=np.array(case), kind=np.array("3dgs"), fused=np.array(False),
             rounded=np.zeros(0, "U1"),
             W=np.array(W), H=np.array(H), kernel_size=np.array(-1.0),
             spec_stats=np.array([[0, 0], [0, 0], [1, 0], [1, 0]], np.int64))
    for k in scenes.INPUT_KEYS + ("viewmatrix", "projmatrix", "campos"):
        if s.get(k) is not None:
            Z["in_" + k] = Z["exp_" + k] = np.ascontiguousarray(s[k], dtype=np.float32)
    for k, v in (("tanfovx", s["tanfovx"]), ("tanfovy", s["tanfovy"]), ("D", s["D"]), ("scale_modifier", s["scale_modifier"])):
        Z["in_" + k] = np.array(v)
    vis = out["radii"] > 0
    for r in ("r1", "r2", "r3"):
        for k in RECORDS:  # the export holds zeros for culled Gaussians
            Z[f"{r}_{k}"] = np.where(vis.reshape((-1,) + (1,) * (geo[k].ndim - 1)), geo[k], 0).astype(geo[k].dtype)
        Z[f"{r}_point_list"], Z[f"{r}_ranges"] = b["point_list"].astype(np.int32), b["ranges"].astype(np.int32)
        Z[f"{r}_n_contrib"], Z[f"{r}_final_T"] = b["n_contrib"].astype(np.int32), b["final_T"]
        Z[f"{r}_planes"] = np.concatenate([out["color"], out["depth"], out["median"], out["opacity"]]).astype(np.float32)
        Z[f"{r}_radii"], Z[f"{r}_R"] = out["radii"], np.array(out["num_rendered"])
        Z[f"{r}_num_binned"] = np.array(int(b["ranges"][:, 1].max()))
    return Z


def _first_stage(Z):
    try:
        judge(Z)
    except StageFailure as e:
        return e.stage, str(e)
    return None, ""


def test_checkers_pass_on_the_oracle_and_name_the_stage_of_a_seeded_fault():
    Z = oracle_npz("A")
    assert _first_stage(Z) == (None, "")
    W, H = int(Z["W"]), int(Z["H"])
    rg, pl = Z["r1_ranges"].astype(np.int64), Z["r1_point_list"]
    lists, _, _ = C64.tile_lists(Z["r1_means2D"], Z["r1_radii"], Z["r1_depths"], W, H)

    # (a) two instances swapped across a tile boundary: the last of tile t and the first of the next non-empty tile,
    # at a boundary where the first one does not belong to the next tile at all
    live = np.nonzero(rg[:, 1] > rg[:, 0])[0]
    t, t2 = next((a, b) for a, b in zip(live[:-1], live[1:]) if int(pl[rg[a, 1] - 1]) not in lists[b])
    F = dict(Z)
    for r in ("r1", "r2", "r3"):
        q = Z[f"{r}_point_list"].copy()
        e = rg[t, 1]
        q[e - 1], q[e] = q[e], q[e - 1]
        F[f"{r}_point_list"] = q
    stage, msg = _first_stage(F)
    assert stage == "scatter+sort", msg
    assert "tiles" in msg and "not theirs" in msg

    # (b) one depth off by 1e-3 in the first forward only
    F = dict(Z)
    d = Z["r1_depths"].copy()
    i = int(np.nonzero(Z["r1_radii"] > 0)[0][7])
    d[i] += np.float32(1e-3)
    F["r1_depths"] = d
    stage, msg = _first_stage(F)
    assert stage == "projection", msg
    assert f"#{i}" in msg and "depths" in msg

    # (c) the ranges shifted by one
    F = dict(Z)
    for r in ("r1", "r2", "r3"):
        q = Z[f"{r}_ranges"].copy()
        q[q[:, 1] > q[:, 0]] += 1
        F[f"{r}_ranges"] = q
    stage, msg = _first_stage(F)
    assert stage == "scan", msg

    # a wrong pixel alone is a compositing failure; a first forward that differs from its re-renders in one plane value
    # that the float64 bound cannot see is still caught, by reproducibility
    F = dict(Z)
    p = Z["r1_planes"].copy()
    for r in ("r1", "r2", "r3"):
        F[f"{r}_planes"] = p
    y, x = np.unravel_index(int(np.argmax(p[7])), p[7].shape)
    p[0, y, x] += np.float32(5e-3)
    stage, msg = _first_stage(F)
    assert stage == "compositing", msg
    F = dict(Z)
    p = Z["r1_planes"].copy()
    p[0, y, x] = np.nextafter(p[0, y, x], np.float32(2))
    F["r1_planes"] = p
    stage, msg = _first_stage(F)
    assert stage == "reproducibility" and "1 pixels in 1 of" in msg, msg

    # an input that is not what the activations give
    F = dict(Z)
    q = Z["in_opacities"].copy()
    q[3] = np.nextafter(q[3], np.float32(2))
    F["in_opacities"] = q
    assert _first_stage(F)[0] == "inputs"


# ---- GPU: one child per case -------------------------------------------------------------------------------------------
CASES = [("materialised", "cfg5"), ("same_stream", "cfg5"), ("same_stream_fused", "cfg5"), ("side_stream_waited", "cfg5"),
         ("non_default_stream", "cfg5"), ("after_allocator_churn", "cfg5"), ("eager_modules", "cfg5"), ("mip", "cfg5"),
         ("surfel", "cfg5"), ("same_stream", "B"), ("same_stream", "cfg1")]


def run_child(case, scene, out):
    env = dict(os.environ)
    for k in ("GSR_FWD_TMA", "GSR_BWD_NSUB", "GSR_SPECULATE", "GSR_TILE_ORDER", "GSR_PRIORITY", "CUDA_MODULE_LOADING"):
        env.pop(k, None)
    if case == "eager_modules":
        env["CUDA_MODULE_LOADING"] = "EAGER"
    child_case = "same_stream" if case == "eager_modules" else case
    # subprocess.run kills the child when the timeout expires: nothing is left running, and nothing is retried
    r = subprocess.run([sys.executable, CHILD, "--case", child_case, "--scene", scene, "--out", out], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, f"{case} / {scene}: the child failed\n{r.stderr[-3000:]}"
    return dict(np.load(out))


@pytest.mark.gpu
@pytest.mark.parametrize("case,scene", CASES, ids=[f"{c}-{s}" for c, s in CASES])
def test_first_forward_stage_by_stage(case, scene, tmp_path):
    Z = run_child(case, scene, str(tmp_path / "state.npz"))
    if case == "eager_modules":
        assert str(Z["module_loading"]) == "EAGER"
    try:
        notes = judge(Z)
    except StageFailure as e:
        raise AssertionError(f"{case} / {scene}: {e}") from None
    vis = int((Z["r1_radii"] > 0).sum())
    assert vis > 0 and int(Z["r1_R"]) > 0
    print(f"\n{case} / {scene}: every stage passed; {vis} of {Z['r1_radii'].shape[0]} Gaussians visible, num_rendered "
          f"{int(Z['r1_R'])}, binned {int(Z['r1_num_binned']) if 'r1_num_binned' in Z else '-'}; notes {notes}")
