"""Python mirror of the reference's pybind11 module `_C`
($RAST/ext.cpp:15-19, $RAST/rasterize_points.cu:35-231): same three functions, same argument order, same
returned tuples -- implemented on top of the C ABI of libgsr_b200.so (include/gsr.h) through ctypes.
PyTorch is only the owner of device memory and of the current stream here.
"""
import ctypes as C
import math
import threading

import torch

from . import _lib
from ._lib import ALLOC, call, ptr as _ptr

# Pipelined (sync-free) forward: opt-in.  In exact mode (default) the forward does one blocking 8-byte
# device->host read of num_rendered to size the binning buffer, like the reference (rasterizer_impl.cu:284).
# In pipelined mode the binning buffer is sized from the high-water mark of earlier views with the same
# (device, P, W, H) and the count is read asynchronously; an overflow is reported by `check_pipeline()` /
# the next forward (async-error semantics, like CUDA errors without `debug` in the reference).
_pipeline = threading.local()
# Exact mode: `binned` is the pinned int64 the library writes the binned count into, `last_binned` its last value.
_exact = threading.local()


def set_pipelined(enabled, slack=1.25, fixed_capacity=None):
    """enabled: sync-free forward.  fixed_capacity: always size the binning buffer for exactly this many tile
    instances and keep NO host-side bookkeeping (no events, no pinned read-back) -- the mode CUDA-graph capture
    needs (gaustudio_b200.graphs); the caller checks `num_rendered <= capacity` on the device side."""
    _pipeline.enabled = bool(enabled)
    _pipeline.fixed = int(fixed_capacity) if fixed_capacity else 0
    _pipeline.slack = float(slack)
    _pipeline.hw = {}
    _pipeline.pending = []
    _pipeline.ring = None   # pinned int64 ring: one slot per in-flight view (no allocation in the hot path)
    _pipeline.slot = 0
    _pipeline.rmax = None   # fixed-capacity mode: device-side running maximum of num_rendered (int64[1])


def _pl():
    if not hasattr(_pipeline, "enabled"):
        set_pipelined(False)
    return _pipeline


_PL_FIELDS = ("enabled", "fixed", "slack", "hw", "pending", "ring", "slot", "rmax")


def pipeline_state():
    """Snapshot of this thread's forward mode (for code that switches it temporarily, e.g. CUDA-graph capture)."""
    pl = _pl()
    return {k: getattr(pl, k) for k in _PL_FIELDS}


def restore_pipeline(state):
    for k in _PL_FIELDS:
        setattr(_pipeline, k, state[k])


def set_tile_order(mode):
    """CTA -> tile order of the per-tile kernels (gsr_set_tile_order): 1 longest first (default), 0 raster, 2 shortest
    first, < 0 back to the default.  Process-wide; returns the previous mode.  Results never depend on it."""
    return int(_lib.lib().gsr_set_tile_order(int(mode)))


def set_speculation(on):
    """Exact-mode speculation of the forward (gsr_set_speculation): True (default) sizes the binning buffer from the
    previous view's count and enqueues the whole forward before blocking on the count read; False is the plain blocking
    read in the middle of the forward; None restores the default.  Process-wide; returns the previous setting
    (None = default).  Results and the returned num_rendered are identical either way."""
    prev = int(_lib.lib().gsr_set_speculation(-1 if on is None else int(bool(on))))
    return None if prev < 0 else bool(prev)


def speculation_stats():
    """(hits, redos): exact-mode forwards whose capacity guess held / that had to re-bin with the exact count."""
    h, r = C.c_int64(0), C.c_int64(0)
    _lib.lib().gsr_speculation_stats(C.byref(h), C.byref(r))
    return int(h.value), int(r.value)


def last_num_binned():
    """Tile instances the most recent EXACT-mode forward on this thread actually binned.  The returned `num_rendered`
    keeps the reference's meaning (sum of the tile-rect areas); (Gaussian, tile) pairs that cannot reach alpha >= 1/255
    on any pixel of the tile are not binned, so this count -- the one that sizes the binning buffer -- is smaller."""
    return int(getattr(_exact, "last_binned", 0))


def fixed_capacity_max():
    """Largest num_rendered any forward needed since fixed-capacity mode was switched on (one blocking read)."""
    pl = _pl()
    return int(pl.rmax.item()) if pl.rmax is not None else 0


def _quantise(r, slack):
    """Binning capacity for a view that needed r instances: slack on top, rounded up to 1 Mi entries so the
    buffer size (and with it the caching allocator's block) stops changing after the first few views."""
    q = 1 << 20
    return ((int(r * slack) + 4096 + q - 1) // q) * q


def check_pipeline(wait=False):
    """Raise if a pipelined forward overflowed its binning capacity.  wait=True drains all pending views."""
    pl = _pl()
    keep = []
    for host, ev, cap, key in pl.pending:
        if wait:
            ev.synchronize()
        if ev.query():
            r = int(host.item())
            pl.hw[key] = max(pl.hw.get(key, 0), _quantise(r, pl.slack))
            if r > cap:
                pl.pending = []
                raise RuntimeError(f"gsr: pipelined forward overflowed its binning capacity ({r} > {cap}); "
                                   "that view's outputs are incomplete -- re-run it")
        else:
            keep.append((host, ev, cap, key))
    pl.pending = keep


_bg_cache = {}


def _bg_on(t, device):
    """gaustudio keeps the background colour on the CPU (vanilla_renderer.py:23).  A per-call `.to(device)` of a
    pageable tensor is a blocking copy that drains the stream, so device copies are cached by value."""
    if t.device == device:
        return t
    key = (tuple(float(v) for v in t.flatten().tolist()), device.index)
    d = _bg_cache.get(key)
    if d is None:
        d = _bg_cache[key] = t.to(device=device, dtype=torch.float32).contiguous()
    return d


def _f32(t, device, name):
    if t is None or t.numel() == 0:
        return t
    if t.dtype is torch.float32 and t.device == device and t.is_contiguous():
        return t  # the common case: nothing to do
    if t.dtype != torch.float32:
        raise RuntimeError(f"{name} must be float32")
    if t.device != device:
        t = t.to(device)
    return t.contiguous()


def _f32_rot(t, device, name):
    """_f32 for the quaternions, which the kernels read as one 16-byte vector per Gaussian (include/gsr.h): a
    contiguous view at a storage offset that is not a multiple of 4 elements is copied to a fresh, aligned tensor."""
    t = _f32(t, device, name)
    if t is not None and t.numel() != 0 and t.data_ptr() % 16 != 0:
        t = t.clone()
    return t


def rasterize_gaussians(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                        viewmatrix, projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh, degree, campos,
                        prefiltered, debug, _fused=None, _kernel_size=None):
    """_fused=(f_dc, f_rest): fused-activation variant (gsr_forward_fused): `opacity`, `scales`, `rotations` are
    then the model's RAW attributes and `sh` / `colors` / `cov3D_precomp` are ignored.
    _kernel_size: the Mip-Splatting projection (gsr_forward_mip); see rasterize_gaussians_mip."""
    if means3D.ndimension() != 2 or means3D.size(1) != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")  # rasterize_points.cu:57-59
    if not means3D.is_cuda:
        raise RuntimeError("gaustudio_b200 runs on CUDA (sm_90a) only; means3D must be a CUDA tensor")
    dev = means3D.device
    P, H, W = means3D.size(0), int(image_height), int(image_width)
    fopt = dict(dtype=torch.float32, device=dev)
    if P == 0:  # rasterize_points.cu:84
        e = torch.empty(0, dtype=torch.uint8, device=dev)
        return (0, torch.zeros(3, H, W, **fopt), torch.zeros(1, H, W, **fopt), torch.zeros(3, H, W, **fopt),
                torch.zeros(1, H, W, **fopt), torch.zeros(0, dtype=torch.int32, device=dev), e, e.clone(), e.clone())
    means3D = _f32(means3D, dev, "means3D"); colors = _f32(colors, dev, "colors_precomp")
    opacity = _f32(opacity, dev, "opacities"); scales = _f32(scales, dev, "scales")
    rotations = _f32_rot(rotations, dev, "rotations"); cov3D_precomp = _f32(cov3D_precomp, dev, "cov3D_precomp")
    viewmatrix = _f32(viewmatrix, dev, "viewmatrix"); projmatrix = _f32(projmatrix, dev, "projmatrix")
    sh = _f32(sh, dev, "shs"); campos = _f32(campos, dev, "campos")
    background = _f32(_bg_on(background, dev), dev, "bg")  # gaustudio passes a CPU tensor
    M = sh.size(1) if sh.numel() != 0 else 0  # rasterize_points.cu:86-90
    if _fused is not None:
        f_dc, f_rest = (_f32(t, dev, "f_dc/f_rest") for t in _fused)
        M = 1 + (f_rest.numel() // (3 * P) if f_rest.numel() else 0)

    planes = torch.empty(8, H, W, **fopt)  # one allocation, four contiguous views
    out_color, out_depth, out_median, out_opacity = planes[0:3], planes[3:4], planes[4:7], planes[7:8]
    radii = torch.empty(P, dtype=torch.int32, device=dev)

    pl = _pl()
    cap, host = 0, None
    key = (dev.index, P, W, H)
    if pl.enabled and pl.fixed:
        cap = pl.fixed
    elif pl.enabled:
        check_pipeline()
        cap = pl.hw.get(key, 0)
        if cap > 0:
            if pl.ring is None:
                pl.ring = torch.zeros(256, dtype=torch.int64).pin_memory()
            if len(pl.pending) >= 200:
                check_pipeline(wait=True)
            host = pl.ring[pl.slot:pl.slot + 1]
            pl.slot = (pl.slot + 1) % 256
    exact = cap == 0
    if exact:  # the library also hands back the binned count (what sizes the binning buffer) through r_host
        if getattr(_exact, "binned", None) is None:
            _exact.binned = torch.zeros(1, dtype=torch.int64).pin_memory()
        host = _exact.binned
    # the three resizable byte tensors of rasterize_points.cu:27-33,74-81: slots 1, 2, 3 = geometry, binning, image
    with _lib.scratch(dev) as slots:
        tail = (float(tan_fovx), float(tan_fovy), int(bool(prefiltered)), _ptr(out_color), _ptr(out_depth),
                _ptr(out_median), _ptr(out_opacity), _ptr(radii), int(bool(debug)), int(cap), _ptr(host))
        if _kernel_size is not None:
            r = call("gsr_forward_mip", dev, ALLOC, 1, ALLOC, 2, ALLOC, 3, P, int(degree), M, _ptr(background), W, H,
                     _ptr(means3D), _ptr(sh), _ptr(colors), _ptr(opacity), _ptr(scales), float(scale_modifier),
                     _ptr(rotations), _ptr(cov3D_precomp), _ptr(viewmatrix), _ptr(projmatrix), _ptr(campos), *tail,
                     float(_kernel_size))
        elif _fused is None:
            r = call("gsr_forward", dev, ALLOC, 1, ALLOC, 2, ALLOC, 3, P, int(degree), M, _ptr(background), W, H,
                     _ptr(means3D), _ptr(sh), _ptr(colors), _ptr(opacity), _ptr(scales), float(scale_modifier),
                     _ptr(rotations), _ptr(cov3D_precomp), _ptr(viewmatrix), _ptr(projmatrix), _ptr(campos), *tail)
        else:
            r = call("gsr_forward_fused", dev, ALLOC, 1, ALLOC, 2, ALLOC, 3, P, int(degree), M, _ptr(background), W,
                     H, _ptr(means3D), _ptr(f_dc), _ptr(f_rest), _ptr(opacity), _ptr(scales), float(scale_modifier),
                     _ptr(rotations), _ptr(viewmatrix), _ptr(projmatrix), _ptr(campos), *tail)
        if pl.enabled and pl.fixed:
            # no host bookkeeping in this mode: the largest count any view needed is tracked on the device (the
            # opaque image buffer starts with num_rendered as a uint64) and read by `fixed_capacity_max()`
            if pl.rmax is None or pl.rmax.device != dev:
                pl.rmax = torch.zeros(1, dtype=torch.int64, device=dev)
            torch.maximum(pl.rmax, slots[3][:8].view(torch.int64), out=pl.rmax)
    if exact:
        _exact.last_binned = int(host[0])  # written by the library before it returned (exact mode synchronises)
    if pl.enabled and not pl.fixed:
        if cap > 0:
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(dev))
            pl.pending.append((host, ev, cap, key))
        else:  # first view of this shape ran in exact mode: seed the high-water mark
            pl.hw[key] = _quantise(_exact.last_binned, pl.slack)
    empty = torch.empty(0, dtype=torch.uint8, device=dev)
    return (int(r), out_color, out_depth, out_median, out_opacity, radii, slots.get(1, empty), slots.get(2, empty),
            slots.get(3, empty))


def rasterize_gaussians_backward(background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp,
                                 viewmatrix, projmatrix, tan_fovx, tan_fovy, dL_dout_color, dL_dout_depth,
                                 dL_dout_median_depth, dL_dout_final_opacity, sh, degree, campos, geomBuffer, R,
                                 binningBuffer, imageBuffer, debug, _mip=None):
    """_mip=(opacities, kernel_size): the backward of the Mip-Splatting projection (gsr_backward_mip)."""
    dev = means3D.device
    P = means3D.size(0)
    H, W = dL_dout_color.size(1), dL_dout_color.size(2)
    M = sh.size(1) if sh.numel() != 0 else 0
    fopt = dict(dtype=torch.float32, device=dev)
    alloc = torch.zeros if P == 0 else torch.empty  # every element is written by the kernels when P > 0
    dL_dmeans3D = alloc(P, 3, **fopt); dL_dmeans2D = alloc(P, 3, **fopt); dL_dcolors = alloc(P, 3, **fopt)
    dL_dopacity = alloc(P, 1, **fopt); dL_dcov3D = alloc(P, 6, **fopt); dL_dsh = alloc(P, M, 3, **fopt)
    dL_dscales = alloc(P, 3, **fopt); dL_drotations = alloc(P, 4, **fopt)
    if P != 0:
        means3D = _f32(means3D, dev, "means3D"); colors = _f32(colors, dev, "colors_precomp")
        scales = _f32(scales, dev, "scales"); rotations = _f32_rot(rotations, dev, "rotations")
        cov3D_precomp = _f32(cov3D_precomp, dev, "cov3D_precomp"); viewmatrix = _f32(viewmatrix, dev, "viewmatrix")
        projmatrix = _f32(projmatrix, dev, "projmatrix"); sh = _f32(sh, dev, "shs"); campos = _f32(campos, dev, "campos")
        background = _f32(_bg_on(background, dev), dev, "bg")
        gc = _f32(dL_dout_color, dev, "dL_dout_color"); gd = _f32(dL_dout_depth, dev, "dL_dout_depth")
        gm = _f32(dL_dout_median_depth, dev, "dL_dout_median_depth")
        go = _f32(dL_dout_final_opacity, dev, "dL_dout_final_opacity")
        radii = radii.contiguous()
        args = (P, int(degree), M, int(R), _ptr(background), W, H, _ptr(means3D), _ptr(sh), _ptr(colors),
                _ptr(scales), float(scale_modifier), _ptr(rotations), _ptr(cov3D_precomp), _ptr(viewmatrix),
                _ptr(projmatrix), _ptr(campos), float(tan_fovx), float(tan_fovy), _ptr(radii), _ptr(geomBuffer),
                _ptr(binningBuffer), _ptr(imageBuffer), _ptr(gc), _ptr(gd), _ptr(gm), _ptr(go),
                _ptr(dL_dmeans2D), None, _ptr(dL_dopacity), _ptr(dL_dcolors), None, _ptr(dL_dmeans3D),
                _ptr(dL_dcov3D), _ptr(dL_dsh), _ptr(dL_dscales), _ptr(dL_drotations), int(bool(debug)))
        if _mip is None:
            call("gsr_backward", dev, *args)
        else:
            opac = _f32(_mip[0], dev, "opacities")
            call("gsr_backward_mip", dev, *args, _ptr(opac), float(_mip[1]))
    return dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dscales, dL_drotations


def rasterize_gaussians_fused_backward(background, means3D, radii, f_dc, f_rest, opacity_logits, log_scales,
                                       raw_rotations, scale_modifier, viewmatrix, projmatrix, tan_fovx, tan_fovy,
                                       dL_dout_color, dL_dout_depth, dL_dout_median_depth, dL_dout_final_opacity,
                                       degree, campos, geomBuffer, R, binningBuffer, imageBuffer, debug):
    """Backward of the fused-activation variant: gradients w.r.t. the RAW attributes
    -> (dL_dmeans2D, dL_dopacity_logit, dL_dmeans3D, dL_df_dc, dL_df_rest, dL_dlog_scale, dL_draw_rot)."""
    dev = means3D.device
    P = means3D.size(0)
    H, W = dL_dout_color.size(1), dL_dout_color.size(2)
    fopt = dict(dtype=torch.float32, device=dev)
    f_dc, f_rest = _f32(f_dc, dev, "f_dc"), _f32(f_rest, dev, "f_rest")
    M = 1 + (f_rest.numel() // (3 * P) if f_rest.numel() else 0)
    d_m3 = torch.empty(P, 3, **fopt); d_m2 = torch.empty(P, 3, **fopt); d_op = torch.empty_like(opacity_logits)
    d_dc = torch.empty_like(f_dc); d_rest = torch.empty_like(f_rest); d_sc = torch.empty(P, 3, **fopt)
    d_rot = torch.empty(P, 4, **fopt)
    means3D = _f32(means3D, dev, "means3D"); opacity_logits = _f32(opacity_logits, dev, "opacity")
    log_scales = _f32(log_scales, dev, "scales"); raw_rotations = _f32_rot(raw_rotations, dev, "rotations")
    viewmatrix = _f32(viewmatrix, dev, "viewmatrix"); projmatrix = _f32(projmatrix, dev, "projmatrix")
    campos = _f32(campos, dev, "campos"); background = _f32(_bg_on(background, dev), dev, "bg")
    gc = _f32(dL_dout_color, dev, "dL_dout_color"); gd = _f32(dL_dout_depth, dev, "dL_dout_depth")
    gm = _f32(dL_dout_median_depth, dev, "dL_dout_median_depth"); go = _f32(dL_dout_final_opacity, dev, "dL_dout_opacity")
    call("gsr_backward_fused", dev, P, int(degree), M, int(R), _ptr(background), W, H, _ptr(means3D), _ptr(f_dc),
         _ptr(f_rest), _ptr(opacity_logits), _ptr(log_scales), float(scale_modifier), _ptr(raw_rotations), _ptr(viewmatrix),
         _ptr(projmatrix), _ptr(campos), float(tan_fovx), float(tan_fovy), _ptr(radii), _ptr(geomBuffer),
         _ptr(binningBuffer), _ptr(imageBuffer), _ptr(gc), _ptr(gd), _ptr(gm), _ptr(go), _ptr(d_m2), _ptr(d_op), None,
         _ptr(d_m3), None, _ptr(d_dc), _ptr(d_rest), _ptr(d_sc), _ptr(d_rot), int(bool(debug)))
    return d_m2, d_op, d_m3, d_dc, d_rest, d_sc, d_rot


def contribution(P, image_height, image_width, geomBuffer, R, binningBuffer, imageBuffer, weight, count, max_weight):
    """Adds one view's contribution statistics (gsr_contribution) into weight float64[P], count int64[P] and
    max_weight float32[P] (contiguous, on the buffers' device).  The buffers and R are those a rasterize_gaussians,
    its fused variant or rasterize_gaussians_mip returned for that view.  No host synchronisation."""
    dev = geomBuffer.device
    for t, dt, name in ((weight, torch.float64, "weight"), (count, torch.int64, "count"),
                        (max_weight, torch.float32, "max_weight")):
        if t.dtype != dt or tuple(t.shape) != (P,) or t.device != dev or not t.is_contiguous():
            raise ValueError(f"contribution: {name} must be a contiguous {dt} tensor of shape ({P},) on {dev}")
    call("gsr_contribution", dev, int(P), int(R), int(image_width), int(image_height), _ptr(geomBuffer),
         _ptr(binningBuffer), _ptr(imageBuffer), _ptr(weight), _ptr(count), _ptr(max_weight))


# ---- Mip-Splatting: gsr_forward_mip / gsr_backward_mip / gsr_mip_filter3d (include/gsr.h) -----------------------------
def _check_kernel_size(kernel_size):
    k = float(kernel_size)
    if not (k >= 0.0 and k < float("inf")):
        raise ValueError(f"kernel_size must be finite and >= 0, got {kernel_size!r}")
    return k


def rasterize_gaussians_mip(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                            viewmatrix, projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh, degree, campos,
                            prefiltered, debug, kernel_size):
    """rasterize_gaussians with the 2D Mip filter of width `kernel_size` in the projection (gsr_forward_mip): the
    splats' opacity is opacity * coef and their covariance cov2D + kernel_size I.  Same returned tuple."""
    return rasterize_gaussians(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                               viewmatrix, projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh, degree, campos,
                               prefiltered, debug, _kernel_size=_check_kernel_size(kernel_size))


def rasterize_gaussians_mip_backward(background, means3D, radii, colors, opacities, scales, rotations, scale_modifier,
                                     cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, dL_dout_color,
                                     dL_dout_depth, dL_dout_median_depth, dL_dout_final_opacity, sh, degree, campos,
                                     geomBuffer, R, binningBuffer, imageBuffer, debug, kernel_size):
    """Backward of rasterize_gaussians_mip (gsr_backward_mip): the tuple of rasterize_gaussians_backward, with the
    opacity gradient w.r.t. the input `opacities`."""
    return rasterize_gaussians_backward(background, means3D, radii, colors, scales, rotations, scale_modifier,
                                        cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, dL_dout_color,
                                        dL_dout_depth, dL_dout_median_depth, dL_dout_final_opacity, sh, degree, campos,
                                        geomBuffer, R, binningBuffer, imageBuffer, debug,
                                        _mip=(opacities, _check_kernel_size(kernel_size)))


def debug_projection_backward_mip(means3D, shs, colors_precomp, opacities, scales, scale_modifier, rotations,
                                  cov3D_precomp, viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, image_height,
                                  image_width, degree, radii, geomBuffer, accum, kernel_size):
    """The Mip projection backward alone on caller-chosen per-Gaussian sums `accum` [P,12] (tests; see
    gsr_debug_projection_backward_mip in include/gsr.h).  geomBuffer holds a rasterize_gaussians_mip forward of the same
    Gaussians and camera.  -> dict of every output (mean2D, conic, opacity, color, depth, mean3D, cov3D, shs, scale,
    rot), each fully written by the kernel."""
    dev = means3D.device
    P, H, W = means3D.size(0), int(image_height), int(image_width)
    M = shs.size(1) if shs is not None and shs.numel() != 0 else 0
    means3D, shs, colors_precomp = _f32(means3D, dev, "means3D"), _f32(shs, dev, "shs"), _f32(colors_precomp, dev, "colors")
    opacities, scales = _f32(opacities, dev, "opacities"), _f32(scales, dev, "scales")
    rotations, cov3D_precomp = _f32_rot(rotations, dev, "rotations"), _f32(cov3D_precomp, dev, "cov3D_precomp")
    viewmatrix, projmatrix = _f32(viewmatrix, dev, "viewmatrix"), _f32(projmatrix, dev, "projmatrix")
    campos, radii = _f32(campos, dev, "campos"), radii.contiguous()
    e = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
    o = dict(mean2D=e(P, 3), conic=e(P, 4), opacity=e(P), color=e(P, 3), depth=e(P), mean3D=e(P, 3), cov3D=e(P, 6),
             shs=e(P, M, 3), scale=e(P, 3), rot=e(P, 4))
    acc = accum.to(dev, torch.float32).contiguous()
    call("gsr_debug_projection_backward_mip", dev,
         P, int(degree), M, W, H, _ptr(means3D), _ptr(shs), _ptr(colors_precomp), _ptr(opacities), _ptr(scales),
         float(scale_modifier), _ptr(rotations), _ptr(cov3D_precomp), _ptr(viewmatrix), _ptr(projmatrix),
         _ptr(campos), float(tan_fovx), float(tan_fovy), _ptr(radii), _ptr(geomBuffer), _ptr(acc), _ptr(o["mean2D"]),
         _ptr(o["conic"]), _ptr(o["opacity"]), _ptr(o["color"]), _ptr(o["depth"]), _ptr(o["mean3D"]),
         _ptr(o["cov3D"]), _ptr(o["shs"]), _ptr(o["scale"]), _ptr(o["rot"]), _check_kernel_size(kernel_size), 0)
    return o


def mip_camera_records(cameras, device):
    """[C,16] float32 camera records of gsr_mip_filter3d: R (row-major Camera.R), T, fx, fy, width, height."""
    rows = []
    for c in cameras:
        fx = c.image_width / (2.0 * math.tan(c.FoVx * 0.5))
        fy = c.image_height / (2.0 * math.tan(c.FoVy * 0.5))
        rows.append([float(v) for v in torch.as_tensor(c.R, dtype=torch.float64).reshape(9)] +
                    [float(v) for v in torch.as_tensor(c.T, dtype=torch.float64).reshape(3)] +
                    [fx, fy, float(c.image_width), float(c.image_height)])
    return torch.tensor(rows, dtype=torch.float32).reshape(-1, 16).to(device)


def mip_filter3d(means3D, cameras):
    """Mip-Splatting's 3D smoothing filter [P] over `cameras` (Camera objects, or a [C,16] tensor of
    mip_camera_records) in one device pass (gsr_mip_filter3d).  Raises ValueError when no camera sees any Gaussian
    (one host synchronisation to read the count)."""
    if not means3D.is_cuda:
        raise RuntimeError("gaustudio_b200 runs on CUDA (sm_90a) only; means3D must be a CUDA tensor")
    dev = means3D.device
    P = means3D.size(0)
    recs = cameras if torch.is_tensor(cameras) else mip_camera_records(cameras, dev)
    recs = _f32(recs, dev, "cameras")
    means3D = _f32(means3D, dev, "means3D")
    out = torch.empty(P, dtype=torch.float32, device=dev)
    scratch = torch.empty(3, dtype=torch.int32, device=dev)
    call("gsr_mip_filter3d", dev, P, _ptr(means3D), int(recs.numel() // 16), _ptr(recs), _ptr(out), _ptr(scratch))
    if P == 0 or int(scratch[2]) == 0:
        raise ValueError("compute_3D_filter: no camera sees any Gaussian")
    return out


# ---- Scaffold-GS: gsr_scaffold_visible / _count / _decode / _decode_backward (include/gsr.h) ----------------------------
def scaffold_visible(means3D, scales, rotations, cov3D_precomp, scale_modifier, viewmatrix, projmatrix, tan_fovx,
                     tan_fovy, image_height, image_width, kernel_size):
    """radii [N] (int32) of Gaussians at `means3D` under the Mip projection of width kernel_size: bit-identical to the
    radii rasterize_gaussians_mip gives them.  scales [N,3] + rotations [N,4], or cov3D_precomp [N,6]."""
    if not means3D.is_cuda:
        raise RuntimeError("gaustudio_b200 runs on CUDA (sm_90a) only; means3D must be a CUDA tensor")
    dev = means3D.device
    N = means3D.size(0)
    radii = torch.empty(N, dtype=torch.int32, device=dev)
    means3D = _f32(means3D, dev, "means3D"); scales = _f32(scales, dev, "scales")
    rotations = _f32_rot(rotations, dev, "rotations"); cov3D_precomp = _f32(cov3D_precomp, dev, "cov3D_precomp")
    viewmatrix = _f32(viewmatrix, dev, "viewmatrix"); projmatrix = _f32(projmatrix, dev, "projmatrix")
    call("gsr_scaffold_visible", dev, N, _ptr(means3D), _ptr(scales), _ptr(rotations), _ptr(cov3D_precomp),
         float(scale_modifier), _ptr(viewmatrix), _ptr(projmatrix), int(image_width), int(image_height), float(tan_fovx),
         float(tan_fovy), _check_kernel_size(kernel_size), _ptr(radii))
    return radii


def scaffold_count(opacity):
    """opacity [Nv,k] (the opacity MLP's output) -> (base [Nv+1] int32, M): exclusive prefix of the offsets kept per
    visible anchor (opacity > 0) and their total, read back to the host (one synchronisation)."""
    dev = opacity.device
    Nv, k = opacity.shape
    opacity = _f32(opacity, dev, "opacity")
    buf = torch.empty(Nv + 1 + (Nv + 1023) // 1024, dtype=torch.int32, device=dev)
    call("gsr_scaffold_count", dev, Nv, k, _ptr(opacity), _ptr(buf), _ptr(buf[Nv + 1:]))
    base = buf[:Nv + 1]
    return base, int(base[Nv])


def scaffold_decode(vis, base, M, anchor, offset, scaling, opacity, color, cov):
    """The kept neural Gaussians, rows anchor-major and offset-minor: (xyz [M,3], rgb [M,3], opacity [M,1],
    scales [M,3], rotations [M,4]).  vis [Nv] int64; anchor [N,3], offset [N,k,3], scaling [N,6] full-size; opacity
    [Nv,k], color [Nv,3k], cov [Nv,7k]; base, M from scaffold_count."""
    dev = anchor.device
    Nv, k = opacity.shape
    e = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
    out = (e(M, 3), e(M, 3), e(M, 1), e(M, 3), e(M, 4))
    ins = [_f32(t, dev, n) for t, n in ((anchor, "anchor"), (offset, "offset"), (scaling, "scaling"),
                                        (opacity, "opacity"), (color, "color"), (cov, "cov"))]
    vis = vis.contiguous()
    if M > 0:
        call("gsr_scaffold_decode", dev, Nv, k, _ptr(vis), _ptr(base), *[_ptr(t) for t in ins], *[_ptr(t) for t in out])
    return out


def scaffold_decode_backward(vis, base, M, offset, scaling, opacity, cov, grads):
    """Backward of scaffold_decode.  grads: the upstream gradients of its five outputs (None: zero).
    -> (d_anchor [N,3], d_offset [N,k,3], d_scaling [N,6], d_opacity [Nv,k], d_color [Nv,3k], d_cov [Nv,7k])."""
    dev = offset.device
    N, k = offset.shape[0], offset.shape[1]
    Nv = opacity.shape[0]
    e = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
    d_anchor, d_offset, d_scaling = e(N, 3), e(N, k, 3), e(N, 6)
    d_op, d_col, d_cov = e(Nv, k), e(Nv, 3 * k), e(Nv, 7 * k)
    offset, scaling = _f32(offset, dev, "offset"), _f32(scaling, dev, "scaling")
    opacity, cov = _f32(opacity, dev, "opacity"), _f32(cov, dev, "cov")
    g = [torch.zeros(M, w, dtype=torch.float32, device=dev) if t is None else _f32(t, dev, "grad")
         for t, w in zip(grads, (3, 3, 1, 3, 4))]
    call("gsr_scaffold_decode_backward", dev,
         N, Nv, k, _ptr(vis.contiguous()), _ptr(base), _ptr(offset), _ptr(scaling), _ptr(opacity), _ptr(cov),
         *[_ptr(t) for t in g], _ptr(d_op), _ptr(d_col), _ptr(d_cov), _ptr(d_anchor), _ptr(d_offset), _ptr(d_scaling))
    return d_anchor, d_offset, d_scaling, d_op, d_col, d_cov


def mark_visible(means3D, viewmatrix, projmatrix):
    dev = means3D.device
    P = means3D.size(0)
    present = torch.zeros(P, dtype=torch.bool, device=dev)
    if P != 0:
        means3D = _f32(means3D, dev, "means3D")
        viewmatrix = _f32(viewmatrix, dev, "viewmatrix"); projmatrix = _f32(projmatrix, dev, "projmatrix")
        call("gsr_mark_visible", dev, P, _ptr(means3D), _ptr(viewmatrix), _ptr(projmatrix), _ptr(present))
    return present


def debug_export(P, W, H, R, geomBuffer, binningBuffer, imageBuffer):
    """Internal state of a forward as named tensors (parity tests; see gsr_debug_export in include/gsr.h)."""
    dev = geomBuffer.device
    T = ((W + 15) // 16) * ((H + 15) // 16)
    o = dict(point_list=torch.zeros(R, dtype=torch.int32, device=dev),
             ranges=torch.zeros(T, 2, dtype=torch.int32, device=dev),
             n_contrib=torch.zeros(H, W, dtype=torch.int32, device=dev),
             final_T=torch.zeros(H, W, device=dev), means2D=torch.zeros(P, 2, device=dev),
             conic_opacity=torch.zeros(P, 4, device=dev), depths=torch.zeros(P, device=dev),
             rgb=torch.zeros(P, 3, device=dev), cov3D=torch.zeros(P, 6, device=dev),
             tiles_touched=torch.zeros(P, dtype=torch.int32, device=dev),
             clamped=torch.zeros(P, 3, dtype=torch.uint8, device=dev))
    call("gsr_debug_export", dev, P, W, H, int(R), _ptr(geomBuffer), _ptr(binningBuffer), _ptr(imageBuffer),
         _ptr(o["point_list"]), _ptr(o["ranges"]), _ptr(o["n_contrib"]), _ptr(o["final_T"]), _ptr(o["means2D"]),
         _ptr(o["conic_opacity"]), _ptr(o["depths"]), _ptr(o["rgb"]), _ptr(o["cov3D"]), _ptr(o["tiles_touched"]),
         _ptr(o["clamped"]))
    # `R` is the reference's num_rendered (rect areas); the sorted list holds the binned instances only
    o["num_binned"] = int(o["ranges"][:, 1].max()) if T else 0
    o["point_list"] = o["point_list"][:o["num_binned"]]
    return o


def debug_accumulator(P, geomBuffer):
    """The compositing backward's per-Gaussian sums [P,12] left in geomBuffer by the last backward on it (tests; see
    gsr_debug_accumulator in include/gsr.h)."""
    dev = geomBuffer.device
    out = torch.zeros(P, 12, device=dev)
    if P == 0:
        return out
    call("gsr_debug_accumulator", dev, int(P), _ptr(geomBuffer), _ptr(out))
    return out


# ---- surfel (2D Gaussian) rasterizer: gsr_surfel_forward / gsr_surfel_backward (include/gsr.h) -------------------------
def rasterize_surfels(background, means3D, colors, opacity, scales, rotations, scale_modifier, viewmatrix, projmatrix,
                      tan_fovx, tan_fovy, image_height, image_width, sh, degree, campos, prefiltered, debug):
    """Forward of the surfel rasterizer -> (num_rendered, color[3,H,W], radii[P], allmap[9,H,W], geomBuffer,
    binningBuffer, imageBuffer).  allmap = {expected depth sum, alpha, normal (3), median depth, distortion,
    median weight, median Gaussian index}; see gsr_surfel_forward."""
    if means3D.ndimension() != 2 or means3D.size(1) != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")
    if not means3D.is_cuda:
        raise RuntimeError("gaustudio_b200 runs on CUDA (sm_90a) only; means3D must be a CUDA tensor")
    dev = means3D.device
    P, H, W = means3D.size(0), int(image_height), int(image_width)
    fopt = dict(dtype=torch.float32, device=dev)
    means3D = _f32(means3D, dev, "means3D"); colors = _f32(colors, dev, "colors_precomp")
    opacity = _f32(opacity, dev, "opacities"); scales = _f32(scales, dev, "scales")
    rotations = _f32_rot(rotations, dev, "rotations")
    viewmatrix = _f32(viewmatrix, dev, "viewmatrix"); projmatrix = _f32(projmatrix, dev, "projmatrix")
    sh = _f32(sh, dev, "shs"); campos = _f32(campos, dev, "campos")
    background = _f32(_bg_on(background, dev), dev, "bg")
    M = sh.size(1) if sh is not None and sh.numel() != 0 else 0
    color = torch.empty(3, H, W, **fopt)
    allmap = torch.empty(9, H, W, **fopt)
    radii = torch.empty(P, dtype=torch.int32, device=dev)
    with _lib.scratch(dev) as slots:
        r = call("gsr_surfel_forward", dev, ALLOC, 1, ALLOC, 2, ALLOC, 3, P, int(degree), M, _ptr(background), W, H,
                 _ptr(means3D), _ptr(sh), _ptr(colors), _ptr(opacity), _ptr(scales), float(scale_modifier), _ptr(rotations),
                 _ptr(viewmatrix), _ptr(projmatrix), _ptr(campos), int(bool(prefiltered)), _ptr(color), _ptr(allmap),
                 _ptr(radii), int(bool(debug)))
    empty = torch.empty(0, dtype=torch.uint8, device=dev)
    return (int(r), color, radii, allmap, slots.get(1, empty), slots.get(2, empty), slots.get(3, empty))


def rasterize_surfels_backward(background, means3D, radii, colors, scales, rotations, scale_modifier, viewmatrix,
                               projmatrix, tan_fovx, tan_fovy, dL_dout_color, dL_dout_allmap, sh, degree, campos,
                               geomBuffer, R, binningBuffer, imageBuffer, debug):
    """Backward of rasterize_surfels -> (dL_dmeans2D[P,3], dL_dcolors[P,3], dL_dopacity[P,1], dL_dmeans3D[P,3],
    dL_dsh[P,M,3], dL_dscales[P,2], dL_drotations[P,4]).  Allmap channels 7 and 8 carry no gradient."""
    dev = means3D.device
    P = means3D.size(0)
    H, W = dL_dout_color.size(1), dL_dout_color.size(2)
    M = sh.size(1) if sh is not None and sh.numel() != 0 else 0
    fopt = dict(dtype=torch.float32, device=dev)
    alloc = torch.zeros if P == 0 else torch.empty  # every element is written by the kernels when P > 0
    d_m2 = alloc(P, 3, **fopt); d_col = alloc(P, 3, **fopt); d_op = alloc(P, 1, **fopt); d_m3 = alloc(P, 3, **fopt)
    d_sh = alloc(P, M, 3, **fopt); d_sc = alloc(P, 2, **fopt); d_rot = alloc(P, 4, **fopt)
    if P != 0:
        means3D = _f32(means3D, dev, "means3D"); scales = _f32(scales, dev, "scales")
        rotations = _f32_rot(rotations, dev, "rotations"); viewmatrix = _f32(viewmatrix, dev, "viewmatrix")
        projmatrix = _f32(projmatrix, dev, "projmatrix"); sh = _f32(sh, dev, "shs"); campos = _f32(campos, dev, "campos")
        background = _f32(_bg_on(background, dev), dev, "bg")
        gc = _f32(dL_dout_color, dev, "dL_dout_color"); gm = _f32(dL_dout_allmap, dev, "dL_dout_allmap")
        call("gsr_surfel_backward", dev, P, int(degree), M, int(R), _ptr(background), W, H, _ptr(means3D), _ptr(sh),
             _ptr(scales), float(scale_modifier), _ptr(rotations), _ptr(viewmatrix), _ptr(projmatrix), _ptr(campos),
             _ptr(geomBuffer), _ptr(binningBuffer), _ptr(imageBuffer), _ptr(gc), _ptr(gm), _ptr(d_m2), _ptr(d_op), _ptr(d_col),
             _ptr(d_m3), _ptr(d_sh), _ptr(d_sc), _ptr(d_rot), int(bool(debug)))
    return d_m2, d_col, d_op, d_m3, d_sh, d_sc, d_rot
