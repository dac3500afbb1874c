"""ctypes binding of libgsr_b200.so -- the C ABI declared in include/gsr.h.

There is NO CPU or PyTorch fallback: if the CUDA library is missing or does not export the ABI, importing
this module raises.  (oracle/ is test infrastructure and is never imported from here.)
"""
import contextlib
import ctypes as C
import os
import threading

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# GSR_LIB selects another build of the same sources (the ring-stress variant of the tests); default: the in-tree library
LIB_PATH = os.environ.get("GSR_LIB") or os.path.join(_HERE, "libgsr_b200.so")

ALLOC_FN = C.CFUNCTYPE(C.c_void_p, C.c_void_p, C.c_size_t)
_P, _I, _F, _L, _D = C.c_void_p, C.c_int, C.c_float, C.c_int64, C.c_double

SIGNATURES = {
    "gsr_abi_version": (_I, []),
    "gsr_last_error": (C.c_char_p, []),
    "gsr_geometry_bytes": (C.c_size_t, [_I]),
    "gsr_image_bytes": (C.c_size_t, [_I, _I]),
    "gsr_binning_bytes": (C.c_size_t, [_L]),
    "gsr_forward": (_L, [ALLOC_FN, _P, ALLOC_FN, _P, ALLOC_FN, _P, _I, _I, _I, _P, _I, _I, _P, _P, _P, _P, _P, _F, _P,
                         _P, _P, _P, _P, _F, _F, _I, _P, _P, _P, _P, _P, _I, _L, _P, _P]),
    "gsr_backward": (_I, [_I, _I, _I, _L, _P, _I, _I, _P, _P, _P, _P, _F, _P, _P, _P, _P, _P, _F, _F, _P, _P, _P, _P,
                          _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _P]),
    "gsr_contribution": (_I, [_I, _L, _I, _I, _P, _P, _P, _P, _P, _P, _P]),
    "gsr_forward_fused": (_L, [ALLOC_FN, _P, ALLOC_FN, _P, ALLOC_FN, _P, _I, _I, _I, _P, _I, _I, _P, _P, _P, _P, _P, _F, _P,
                               _P, _P, _P, _F, _F, _I, _P, _P, _P, _P, _P, _I, _L, _P, _P]),
    "gsr_backward_fused": (_I, [_I, _I, _I, _L, _P, _I, _I, _P, _P, _P, _P, _P, _F, _P, _P, _P, _P, _F, _F, _P, _P, _P,
                                _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _P]),
    "gsr_mark_visible": (_I, [_I, _P, _P, _P, _P, _P]),
    "gsr_depth2normal": (_I, [_P, _I, _I, _F, _F, _F, _F, _F, _F, _P, _P, _P]),
    "gsr_depth2point": (_I, [_P, _I, _I, _F, _F, _F, _F, _P, _P, _P]),
    "gsr_masked_bilateral": (_I, [_P, _P, _I, _I, _I, _F, _F, _P, _P, _P, _P]),
    "gsr_extract_normals": (_I, [_P, _P, _P, _P, _I, _I, _F, _F, _F, _F, _P, _F, _F, _P, _P, _P, _P]),
    "gsr_normal_fusion_pass": (_I, [_L, _P, _P, _P, _I, _P, _F, _F, _F, _P, _F, _P, _P, _P, _P]),
    "gsr_normal_fusion_mean": (_I, [_I, _P, _P, _P, _P]),
    "gsr_knn_grid": (_I, [_I, _I, _P, _P, _P, _P, _P, _P]),
    "gsr_tsdf_bytes": (C.c_size_t, [_L]),
    "gsr_tsdf_init": (_I, [_P, _L, _D, _D, _P]),
    "gsr_tsdf_integrate": (_I, [_P, _L, _L, _P, _P, _D, _D, _D, _P]),
    "gsr_tsdf_extract": (_L, [_P, _L, _D, ALLOC_FN, _P, ALLOC_FN, _P, ALLOC_FN, _P, _P, _P]),
    "gsr_tsdf_export": (_L, [_P, _L, ALLOC_FN, _P, _P, _P, _P, _P]),
    "gsr_mesh_face_components": (_I, [_L, _P, _L, ALLOC_FN, _P, _P, _P]),
    "gsr_sap_normalize": (_I, [_L, _P, ALLOC_FN, _P, _P, _P, _P]),
    "gsr_sap_splat": (_I, [_L, _P, _P, _I, ALLOC_FN, _P, _P, _P]),
    "gsr_sap_spectral": (_I, [_I, _D, _P, _P, _P]),
    "gsr_sap_shift_scale": (_I, [_L, _P, _I, _P, ALLOC_FN, _P, _P, _P]),
    "gsr_sap_marching_cubes": (_L, [_I, _P, _P, ALLOC_FN, _P, ALLOC_FN, _P, ALLOC_FN, _P, _P, _P]),
    "gsr_clean_knn": (_I, [_L, _P, _I, ALLOC_FN, _P, _P, _P, _P]),
    "gsr_clean_statistical": (_I, [_L, _P, _I, _D, ALLOC_FN, _P, _P, _P, _P, _P]),
    "gsr_clean_normal": (_I, [_L, _P, _P, _I, _D, ALLOC_FN, _P, _P, _P, _P]),
    "gsr_dist2": (_I, [_L, _P, ALLOC_FN, _P, _P, _P]),
    "gsr_normal2rotation": (_I, [_L, _P, _P, _P]),
    "gsr_mesh_vertex_normals": (_I, [_L, _P, _L, _P, ALLOC_FN, _P, _P, _P]),
    "gsr_mesh_gaussians": (_I, [_L, _I, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "gsr_voxelize": (_L, [_L, _P, _L, _P, _I, _D, ALLOC_FN, _P, _P, _P, _P, _P, _P]),
    "gsr_voxel_colors": (_I, [_L, _P, _P, _P, _I, _D, _P, _P, _P, _P, _P]),
    "gsr_hull_carve": (_I, [_I, _D, _D, _D, _D, _I, _P, _P, _P, _P, _P]),
    "gsr_hull_marching_cubes": (_L, [_I, _P, _D, _D, _D, _D, _D, ALLOC_FN, _P, ALLOC_FN, _P, ALLOC_FN, _P, _P,
                                       _P]),
    "gsr_mesh_raster_bytes": (C.c_size_t, [_L, _L, _I, _I]),
    "gsr_mesh_rasterize": (_I, [_L, _P, _L, _P, _P, _D, _D, _D, _D, _D, _I, _I, _P, C.c_size_t, _P, _P, _P]),
    "gsr_mesh_shade": (_I, [_L, _P, _L, _P, _P, _D, _D, _D, _D, _I, _I, _P, _P, _P, _P, _P, _P]),
    "gsr_mesh_texture_view": (_I, [_L, _P, _L, _P, _P, _D, _D, _D, _D, _I, _I, _P, _P, _I, _P, _P, _P, _P, _P]),
    "gsr_surfel_geometry_bytes": (C.c_size_t, [_I]),
    "gsr_surfel_image_bytes": (C.c_size_t, [_I, _I]),
    "gsr_surfel_forward": (_L, [ALLOC_FN, _P, ALLOC_FN, _P, ALLOC_FN, _P, _I, _I, _I, _P, _I, _I, _P, _P, _P, _P, _P, _F,
                                _P, _P, _P, _P, _I, _P, _P, _P, _I, _P]),
    "gsr_surfel_backward": (_I, [_I, _I, _I, _L, _P, _I, _I, _P, _P, _P, _F, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P,
                                 _P, _P, _P, _P, _P, _I, _P]),
    "gsr_adam_step": (_I, [_I, _P, _D, _D, _D, _L, _I, _F, _I, _P]),
    "gsr_set_tile_order": (_I, [_I]),
    "gsr_set_speculation": (_I, [_I]),
    "gsr_speculation_stats": (_I, [_P, _P]),
    "gsr_profile_enable": (_I, [_I]),
    "gsr_profile_read": (_I, [_P, _P]),
    "gsr_debug_export": (_I, [_I, _I, _I, _L, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "gsr_debug_accumulator": (_I, [_I, _P, _P, _P]),
    "gsr_debug_projection_backward": (_I, [_I, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _F, _P, _P, _P, _P, _P,
                                           _F, _F, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _P]),
    "gsr_forward_mip": (_L, [ALLOC_FN, _P, ALLOC_FN, _P, ALLOC_FN, _P, _I, _I, _I, _P, _I, _I, _P, _P, _P, _P, _P, _F, _P,
                             _P, _P, _P, _P, _F, _F, _I, _P, _P, _P, _P, _P, _I, _L, _P, _F, _P]),
    "gsr_backward_mip": (_I, [_I, _I, _I, _L, _P, _I, _I, _P, _P, _P, _P, _F, _P, _P, _P, _P, _P, _F, _F, _P, _P, _P, _P,
                              _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _P, _F, _P]),
    "gsr_debug_projection_backward_mip": (_I, [_I, _I, _I, _I, _I, _P, _P, _P, _P, _P, _F, _P, _P, _P, _P, _P, _F, _F,
                                               _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _F, _I, _P]),
    "gsr_mip_filter3d": (_I, [_I, _P, _I, _P, _P, _P, _P]),
    "gsr_scaffold_visible": (_I, [_I, _P, _P, _P, _P, _F, _P, _P, _I, _I, _F, _F, _F, _P, _P]),
    "gsr_scaffold_count": (_I, [_I, _I, _P, _P, _P, _P]),
    "gsr_scaffold_decode": (_I, [_I, _I, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "gsr_scaffold_decode_backward": (_I, [_I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P,
                                          _P, _P]),
    "gsr_densify_stats": (_I, [_I, _P, _P, _P, _P, _P, _P]),
    "gsr_densify_count": (_I, [_I, _I, _P, _P, _P, _P, _F, _F, _F, _I, _F, _P, _P]),
    "gsr_densify_apply": (_I, [_I, _I, _P, _I, _I, _I, _I, _P, _I, _P, _P]),
    "gsr_ssim_scratch_bytes": (C.c_size_t, [_L, _I, _I]),
    "gsr_ssim_forward": (_I, [_L, _I, _I, _P, _P, _P, _P, _P, _P]),
    "gsr_ssim_backward": (_I, [_L, _I, _I, _P, _P, _P, _P, _P, _P]),
    "gsr_normal_consistency_scratch_bytes": (C.c_size_t, [_I, _I]),
    "gsr_normal_consistency_forward": (_I, [_I, _I, _P, _P, _P, _P, _F, _F, _F, _F, _P, _P, _P]),
    "gsr_normal_consistency_backward": (_I, [_I, _I, _P, _P, _P, _P, _F, _F, _F, _F, _P, _P, _P, _P]),
}

_lib = None


def ensure_built():
    """Build the library in-tree if the sources are newer (needs nvcc; a no-op on a box that got the .so)."""
    from . import build
    try:
        return build.build_library()
    except Exception:
        if os.path.exists(LIB_PATH):
            return LIB_PATH
        raise


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            ensure_built()
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} not found: run `python -c 'import __graft_entry__ as g; g.build()'`. "
                              "gaustudio_b200 has no CPU / PyTorch fallback.")
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(l, name)  # AttributeError if the ABI is incomplete
            fn.restype = res
            fn.argtypes = args
        if l.gsr_abi_version() != 1:
            raise ImportError("libgsr_b200.so ABI version mismatch")
        _lib = l
    return _lib


def last_error():
    return lib().gsr_last_error().decode()


# ---- host helpers shared by every module that calls the library ----------------------------------------------------
def ptr(t):
    """Device address of a contiguous tensor as a plain int (ctypes converts it for a c_void_p parameter without an
    intermediate object); None (NULL) for an absent / empty tensor."""
    if t is None or t.numel() == 0:
        return None
    return t.data_ptr()


def stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


class on_device:
    """`with torch.cuda.device(dev)` only when `dev` is not already current (the context manager costs ~10 us)."""

    def __init__(self, dev):
        self.ctx = None if torch.cuda.current_device() == dev.index else torch.cuda.device(dev)

    def __enter__(self):
        if self.ctx is not None:
            self.ctx.__enter__()

    def __exit__(self, *exc):
        if self.ctx is not None:
            self.ctx.__exit__(*exc)


def call(name, dev, *args):
    """Entry point `name` of include/gsr.h on `dev`'s current stream (every device entry takes it as its last
    argument); a negative result raises with the library's error text."""
    with on_device(dev):
        r = getattr(lib(), name)(*args, stream(dev))
    if r < 0:
        raise RuntimeError(f"{name} failed: {last_error()}")
    return r


# Scratch of the entries that size their own buffers (gsr_alloc_fn).  ONE persistent callback serves every call: the
# `user` value the caller passed selects the slot of the call in flight on this thread, so no ctypes thunk is created
# per call, and the buffers are plain dict entries (freed by reference counting as soon as the caller drops them; no
# object <-> callback cycle).
_scratch = threading.local()


def _alloc(user, nbytes):
    t = torch.empty(int(nbytes), dtype=torch.uint8, device=_scratch.device)
    _scratch.slots[user] = t
    return t.data_ptr()


ALLOC = ALLOC_FN(_alloc)


@contextlib.contextmanager
def scratch(dev):
    """-> dict slot -> uint8 tensor on `dev`, filled by ALLOC during the `with`; the thread lets go of it on exit."""
    _scratch.device, _scratch.slots = dev, {}
    try:
        yield _scratch.slots
    finally:
        _scratch.slots = None


def call_mesh(name, dev, *args):
    """Entry point `name` that returns a mesh: `args` are its arguments before the trailing (scratch_alloc, scratch_user,
    vertex_alloc, vertex_user, face_alloc, face_user, n_faces).  -> (vertices [V,3] float32, faces [F,3] int64) on
    `dev`, both [0,3] when there is no mesh."""
    nf = C.c_int64(0)
    with scratch(dev) as bufs:
        nv = call(name, dev, *args, ALLOC, 1, ALLOC, 2, ALLOC, 3, C.byref(nf))
    F = nf.value
    v = bufs[2].view(torch.float32).reshape(nv, 3) if nv else torch.empty(0, 3, device=dev)
    f = bufs[3].view(torch.int64).reshape(F, 3) if F else torch.empty(0, 3, dtype=torch.int64, device=dev)
    return v, f
