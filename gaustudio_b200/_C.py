"""Python mirror of the reference's pybind11 module `_C`
($RAST/ext.cpp:15-19, $RAST/rasterize_points.cu:35-231): same three functions, same argument order, same
returned tuples -- implemented on top of the C ABI of libgsr_b200.so (include/gsr.h) through ctypes.
PyTorch is only the owner of device memory and of the current stream here.
"""
import ctypes as C
import threading

import torch

from . import _lib

# Pipelined (sync-free) forward: opt-in.  In exact mode (default) the forward does one blocking 8-byte
# device->host read of num_rendered to size the binning buffer, like the reference (rasterizer_impl.cu:284).
# In pipelined mode the binning buffer is sized from the high-water mark of earlier views with the same
# (device, P, W, H) and the count is read asynchronously; an overflow is reported by `check_pipeline()` /
# the next forward (async-error semantics, like CUDA errors without `debug` in the reference).
_pipeline = threading.local()


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
    return int(getattr(_scratch, "last_binned", 0))


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


def _ptr(t):
    """Device address of a contiguous tensor as a plain int (ctypes converts it for a c_void_p parameter without an
    intermediate object); None (NULL) for an absent / empty tensor."""
    if t is None or t.numel() == 0:
        return None
    return t.data_ptr()


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


class _on_device:
    """`with torch.cuda.device(dev)` only when `dev` is not already current (the context manager costs ~10 us)."""

    def __init__(self, dev):
        self.ctx = None if torch.cuda.current_device() == dev.index else torch.cuda.device(dev)

    def __enter__(self):
        if self.ctx is not None:
            self.ctx.__enter__()

    def __exit__(self, *exc):
        if self.ctx is not None:
            self.ctx.__exit__(*exc)


# The three resizable byte tensors of rasterize_points.cu:27-33,74-81.  ONE persistent ABI callback serves every
# call: `user` (1, 2, 3 = geometry, binning, image) selects the slot of the forward in flight on this thread, so no
# ctypes thunk is created per view, and the buffers are plain list entries (freed by reference counting as soon as
# autograd drops them, like the reference's tensors; no object <-> callback cycle).
_scratch = threading.local()


def _alloc(user, nbytes):
    t = torch.empty(int(nbytes), dtype=torch.uint8, device=_scratch.device)
    _scratch.slots[user] = t
    return t.data_ptr()


_ALLOC = _lib.ALLOC_FN(_alloc)


def rasterize_gaussians(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                        viewmatrix, projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh, degree, campos,
                        prefiltered, debug, _fused=None):
    """_fused=(f_dc, f_rest): fused-activation variant (gsr_forward_fused): `opacity`, `scales`, `rotations` are
    then the model's RAW attributes and `sh` / `colors` / `cov3D_precomp` are ignored."""
    if means3D.ndimension() != 2 or means3D.size(1) != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")  # rasterize_points.cu:57-59
    if not means3D.is_cuda:
        raise RuntimeError("gaustudio_b200 runs on CUDA (sm_90a) only; means3D must be a CUDA tensor")
    L = _lib.lib()
    dev = means3D.device
    P, H, W = means3D.size(0), int(image_height), int(image_width)
    fopt = dict(dtype=torch.float32, device=dev)
    if P == 0:  # rasterize_points.cu:84
        e = torch.empty(0, dtype=torch.uint8, device=dev)
        return (0, torch.zeros(3, H, W, **fopt), torch.zeros(1, H, W, **fopt), torch.zeros(3, H, W, **fopt),
                torch.zeros(1, H, W, **fopt), torch.zeros(0, dtype=torch.int32, device=dev), e, e.clone(), e.clone())
    means3D = _f32(means3D, dev, "means3D"); colors = _f32(colors, dev, "colors_precomp")
    opacity = _f32(opacity, dev, "opacities"); scales = _f32(scales, dev, "scales")
    rotations = _f32(rotations, dev, "rotations"); cov3D_precomp = _f32(cov3D_precomp, dev, "cov3D_precomp")
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
    _scratch.device, _scratch.slots = dev, {}

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
        if getattr(_scratch, "binned", None) is None:
            _scratch.binned = torch.zeros(1, dtype=torch.int64).pin_memory()
        host = _scratch.binned
    with _on_device(dev):
        stream = torch.cuda.current_stream(dev)
        tail = (float(tan_fovx), float(tan_fovy), int(bool(prefiltered)), _ptr(out_color), _ptr(out_depth),
                _ptr(out_median), _ptr(out_opacity), _ptr(radii), int(bool(debug)), int(cap),
                host.data_ptr() if host is not None else None, stream.cuda_stream)
        if _fused is None:
            r = L.gsr_forward(_ALLOC, 1, _ALLOC, 2, _ALLOC, 3, P, int(degree), M, _ptr(background), W, H,
                              _ptr(means3D), _ptr(sh), _ptr(colors), _ptr(opacity), _ptr(scales),
                              float(scale_modifier), _ptr(rotations), _ptr(cov3D_precomp), _ptr(viewmatrix),
                              _ptr(projmatrix), _ptr(campos), *tail)
        else:
            r = L.gsr_forward_fused(_ALLOC, 1, _ALLOC, 2, _ALLOC, 3, P, int(degree), M, _ptr(background),
                                    W, H, _ptr(means3D), _ptr(f_dc), _ptr(f_rest), _ptr(opacity), _ptr(scales),
                                    float(scale_modifier), _ptr(rotations), _ptr(viewmatrix), _ptr(projmatrix),
                                    _ptr(campos), *tail)
        if r < 0:
            raise RuntimeError("gsr_forward failed: " + _lib.last_error())
        if pl.enabled and pl.fixed:
            # no host bookkeeping in this mode: the largest count any view needed is tracked on the device (the
            # opaque image buffer starts with num_rendered as a uint64) and read by `fixed_capacity_max()`
            if pl.rmax is None or pl.rmax.device != dev:
                pl.rmax = torch.zeros(1, dtype=torch.int64, device=dev)
            torch.maximum(pl.rmax, _scratch.slots[3][:8].view(torch.int64), out=pl.rmax)
        if exact:
            _scratch.last_binned = int(host[0])  # written by the library before it returned (exact mode synchronises)
        if pl.enabled and not pl.fixed:
            if cap > 0:
                ev = torch.cuda.Event()
                ev.record(stream)
                pl.pending.append((host, ev, cap, key))
            else:  # first view of this shape ran in exact mode: seed the high-water mark
                pl.hw[key] = _quantise(_scratch.last_binned, pl.slack)
    slots, _scratch.slots = _scratch.slots, None
    empty = torch.empty(0, dtype=torch.uint8, device=dev)
    return (int(r), out_color, out_depth, out_median, out_opacity, radii, slots.get(1, empty), slots.get(2, empty),
            slots.get(3, empty))


def rasterize_gaussians_backward(background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp,
                                 viewmatrix, projmatrix, tan_fovx, tan_fovy, dL_dout_color, dL_dout_depth,
                                 dL_dout_median_depth, dL_dout_final_opacity, sh, degree, campos, geomBuffer, R,
                                 binningBuffer, imageBuffer, debug):
    L = _lib.lib()
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
        scales = _f32(scales, dev, "scales"); rotations = _f32(rotations, dev, "rotations")
        cov3D_precomp = _f32(cov3D_precomp, dev, "cov3D_precomp"); viewmatrix = _f32(viewmatrix, dev, "viewmatrix")
        projmatrix = _f32(projmatrix, dev, "projmatrix"); sh = _f32(sh, dev, "shs"); campos = _f32(campos, dev, "campos")
        background = _f32(_bg_on(background, dev), dev, "bg")
        gc = _f32(dL_dout_color, dev, "dL_dout_color"); gd = _f32(dL_dout_depth, dev, "dL_dout_depth")
        gm = _f32(dL_dout_median_depth, dev, "dL_dout_median_depth")
        go = _f32(dL_dout_final_opacity, dev, "dL_dout_final_opacity")
        radii = radii.contiguous()
        with _on_device(dev):
            stream = torch.cuda.current_stream(dev)
            rc = L.gsr_backward(P, int(degree), M, int(R), _ptr(background), W, H, _ptr(means3D), _ptr(sh),
                                _ptr(colors), _ptr(scales), float(scale_modifier), _ptr(rotations),
                                _ptr(cov3D_precomp), _ptr(viewmatrix), _ptr(projmatrix), _ptr(campos), float(tan_fovx),
                                float(tan_fovy), _ptr(radii), _ptr(geomBuffer), _ptr(binningBuffer),
                                _ptr(imageBuffer), _ptr(gc), _ptr(gd), _ptr(gm), _ptr(go), _ptr(dL_dmeans2D), None,
                                _ptr(dL_dopacity), _ptr(dL_dcolors), None, _ptr(dL_dmeans3D), _ptr(dL_dcov3D),
                                _ptr(dL_dsh), _ptr(dL_dscales), _ptr(dL_drotations), int(bool(debug)),
                                stream.cuda_stream)
        if rc < 0:
            raise RuntimeError("gsr_backward failed: " + _lib.last_error())
    return dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dscales, dL_drotations


def rasterize_gaussians_fused_backward(background, means3D, radii, f_dc, f_rest, opacity_logits, log_scales,
                                       raw_rotations, scale_modifier, viewmatrix, projmatrix, tan_fovx, tan_fovy,
                                       dL_dout_color, dL_dout_depth, dL_dout_median_depth, dL_dout_final_opacity,
                                       degree, campos, geomBuffer, R, binningBuffer, imageBuffer, debug):
    """Backward of the fused-activation variant: gradients w.r.t. the RAW attributes
    -> (dL_dmeans2D, dL_dopacity_logit, dL_dmeans3D, dL_df_dc, dL_df_rest, dL_dlog_scale, dL_draw_rot)."""
    L = _lib.lib()
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
    log_scales = _f32(log_scales, dev, "scales"); raw_rotations = _f32(raw_rotations, dev, "rotations")
    viewmatrix = _f32(viewmatrix, dev, "viewmatrix"); projmatrix = _f32(projmatrix, dev, "projmatrix")
    campos = _f32(campos, dev, "campos"); background = _f32(_bg_on(background, dev), dev, "bg")
    gc = _f32(dL_dout_color, dev, "dL_dout_color"); gd = _f32(dL_dout_depth, dev, "dL_dout_depth")
    gm = _f32(dL_dout_median_depth, dev, "dL_dout_median_depth"); go = _f32(dL_dout_final_opacity, dev, "dL_dout_opacity")
    with _on_device(dev):
        stream = torch.cuda.current_stream(dev)
        rc = L.gsr_backward_fused(P, int(degree), M, int(R), _ptr(background), W, H, _ptr(means3D), _ptr(f_dc),
                                  _ptr(f_rest), _ptr(opacity_logits), _ptr(log_scales), float(scale_modifier),
                                  _ptr(raw_rotations), _ptr(viewmatrix), _ptr(projmatrix), _ptr(campos), float(tan_fovx),
                                  float(tan_fovy), _ptr(radii), _ptr(geomBuffer), _ptr(binningBuffer), _ptr(imageBuffer),
                                  _ptr(gc), _ptr(gd), _ptr(gm), _ptr(go), _ptr(d_m2), _ptr(d_op), None, _ptr(d_m3),
                                  None, _ptr(d_dc), _ptr(d_rest), _ptr(d_sc), _ptr(d_rot), int(bool(debug)),
                                  stream.cuda_stream)
    if rc < 0:
        raise RuntimeError("gsr_backward_fused failed: " + _lib.last_error())
    return d_m2, d_op, d_m3, d_dc, d_rest, d_sc, d_rot


def mark_visible(means3D, viewmatrix, projmatrix):
    L = _lib.lib()
    dev = means3D.device
    P = means3D.size(0)
    present = torch.zeros(P, dtype=torch.bool, device=dev)
    if P != 0:
        means3D = _f32(means3D, dev, "means3D")
        viewmatrix = _f32(viewmatrix, dev, "viewmatrix"); projmatrix = _f32(projmatrix, dev, "projmatrix")
        with torch.cuda.device(dev):
            rc = L.gsr_mark_visible(P, _ptr(means3D), _ptr(viewmatrix), _ptr(projmatrix), present.data_ptr(),
                                    torch.cuda.current_stream(dev).cuda_stream)
        if rc < 0:
            raise RuntimeError("gsr_mark_visible failed: " + _lib.last_error())
    return present


def debug_export(P, W, H, R, geomBuffer, binningBuffer, imageBuffer):
    """Internal state of a forward as named tensors (parity tests; see gsr_debug_export in include/gsr.h)."""
    L = _lib.lib()
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
    with torch.cuda.device(dev):
        rc = L.gsr_debug_export(P, W, H, int(R), _ptr(geomBuffer), _ptr(binningBuffer), _ptr(imageBuffer),
                                _ptr(o["point_list"]), _ptr(o["ranges"]), _ptr(o["n_contrib"]), _ptr(o["final_T"]),
                                _ptr(o["means2D"]), _ptr(o["conic_opacity"]), _ptr(o["depths"]), _ptr(o["rgb"]),
                                _ptr(o["cov3D"]), _ptr(o["tiles_touched"]), _ptr(o["clamped"]),
                                torch.cuda.current_stream(dev).cuda_stream)
    if rc < 0:
        raise RuntimeError("gsr_debug_export failed: " + _lib.last_error())
    # `R` is the reference's num_rendered (rect areas); the sorted list holds the binned instances only
    o["num_binned"] = int(o["ranges"][:, 1].max()) if T else 0
    o["point_list"] = o["point_list"][:o["num_binned"]]
    return o
