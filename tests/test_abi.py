"""The C-ABI library loads and exports every symbol include/gsr.h declares (no compute without a GPU)."""
import ctypes
import os
import re

import pytest

from gaustudio_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "gsr.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    names = set(re.findall(r"\b(gsr_[a-z0-9_]+)\s*\(", src))
    names.discard("gsr_alloc_fn")
    return names


def _type_class(decl):
    """'pointer' for any pointer type, otherwise the C type itself (int, float, double, int64_t, size_t, gsr_alloc_fn)."""
    return "pointer" if "*" in decl else decl.replace("const", "").strip()


def _prototypes():
    """name -> (result type class, [(type class, parameter name), ...]) for every function include/gsr.h declares."""
    src = open(os.path.join(ROOT, "include", "gsr.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    src = re.sub(r"^\s*#.*$", "", src, flags=re.M)
    protos = {}
    for ret, name, params in re.findall(r"([A-Za-z_][\w\s*]*?)\s*\b(gsr_\w+)\s*\(([^()]*)\)\s*;", src):
        args = [re.fullmatch(r"(.*?)(\w+)", p.strip()).groups() for p in params.split(",") if p.strip() != "void"]
        protos[name] = (_type_class(ret), [(_type_class(t), n) for t, n in args])
    return protos


def test_every_declared_symbol_is_exported_and_bound():
    names = _declared()
    assert {"gsr_forward", "gsr_backward", "gsr_mark_visible", "gsr_depth2normal", "gsr_last_error"} <= names
    raw = ctypes.CDLL(_lib.LIB_PATH)
    for n in names:
        assert hasattr(raw, n), f"{n} declared in include/gsr.h but not exported"
        assert n in _lib.SIGNATURES, f"{n} has no ctypes signature"
    assert set(_lib.SIGNATURES) <= names


def test_ctypes_signatures_match_the_header():
    """Every _lib.SIGNATURES entry has its prototype's result and argument count, with the same type class at every
    position, so no ctypes call site can shift an argument into its neighbour's slot unnoticed."""
    protos = _prototypes()
    assert set(protos) == _declared()
    C = ctypes
    cls = {C.c_void_p: "pointer", C.c_char_p: "pointer", C.c_int: "int", C.c_float: "float", C.c_double: "double",
           C.c_int64: "int64_t", C.c_size_t: "size_t", _lib.ALLOC_FN: "gsr_alloc_fn"}
    for name, (res, args) in _lib.SIGNATURES.items():
        ret, params = protos[name]
        assert cls[res] == ret, name
        assert [cls[t] for t in args] == [c for c, _ in params], name


def test_host_only_entry_points():
    L = _lib.lib()
    assert L.gsr_abi_version() == 1
    g1, g2 = L.gsr_geometry_bytes(1000), L.gsr_geometry_bytes(2000)
    assert 0 < g1 < g2 and g2 < 2 * g1 + 8192
    assert L.gsr_geometry_bytes(1_000_000) < 144 * 1_000_000  # ~141 B per Gaussian of forward+backward state
    i1 = L.gsr_image_bytes(1920, 1080)
    assert 8 * 1920 * 1080 <= i1 < 9 * 1920 * 1080 + 1_000_000
    assert L.gsr_binning_bytes(0) >= 0 and 20 * 2**20 <= L.gsr_binning_bytes(10**6) < 21 * 2**20  # 20 B per instance, 1 Mi granules
    assert L.gsr_binning_bytes(2**20 + 1) > L.gsr_binning_bytes(2**20) == L.gsr_binning_bytes(2**20 - 5)
    assert isinstance(_lib.last_error(), str)


def test_speculation_switch_round_trip():
    """gsr_set_speculation / gsr_speculation_stats are host-only: the switch returns the previous setting (None =
    default), the counters start at zero in a process that has rendered nothing, and the default build carries no
    experimental cluster-scan kernel (DESIGN.md 3.5)."""
    from gaustudio_b200 import _C
    prev = _C.set_speculation(False)
    try:
        assert _C.set_speculation(True) is False
        assert _C.set_speculation(None) is True
        assert _C.set_speculation(None) is None
        hits, redos = _C.speculation_stats()
        assert hits >= 0 and redos >= 0
    finally:
        _C.set_speculation(prev)
    blob = open(_lib.LIB_PATH, "rb").read()
    assert b"k_tile_scan_cluster" not in blob


class _Off:
    """Argument override: the parameter's default (16-byte aligned) fake address moved by `n` bytes."""

    def __init__(self, n):
        self.n = n


_FAILING_ALLOC = _lib.ALLOC_FN(lambda user, n: None)


def _call(entry, **kw):
    """Calls a C entry point with its arguments given by their names in include/gsr.h.  Defaults: P = 10, D = 0, M = 1,
    32 x 32 pixels, other ints 0, floats 0.5, an allocator that always fails, NULL user data / r_host / stream, and a
    distinct 16-byte aligned fake device address for every other pointer (never dereferenced: every call made with
    them must be refused before the library touches memory or calls CUDA)."""
    ints = {"P": 10, "D": 0, "M": 1, "width": 32, "height": 32}
    args = []
    for i, (cls, name) in enumerate(_prototypes()[entry][1]):
        if name in kw:
            v = kw.pop(name)
        elif cls == "pointer":
            v = None if name in ("stream", "r_host") or name.endswith("_user") else _Off(0)
        else:
            v = {"gsr_alloc_fn": _FAILING_ALLOC, "float": 0.5}.get(cls, ints.get(name, 0))
        args.append((1 << 20) + 4096 * i + v.n if isinstance(v, _Off) else v)
    assert not kw, f"{entry} has no parameter {sorted(kw)}"
    return getattr(_lib.lib(), entry)(*args)


POSITIVE = "gsr_forward: P, width and height must be positive"
SH_MISMATCH = "gsr_forward: sh degree / coefficient count mismatch"
TOO_LARGE = "gsr_forward: image too large"
NO_SCRATCH = "gsr_forward: scratch allocation failed"
NO_STATE = "gsr_backward: missing state buffers"
NO_BACKGROUND = "gsr_backward: background must be a device pointer (backward.cu:586 reads it)"
NO_SCALES = "gsr_backward: scales and rotations are required when cov3D_precomp is NULL"
BWD_ALIGN = "gsr_backward: rotations, dL_drot and dL_dconic must be 16-byte aligned"
NO_ACCUM = "gsr_debug_projection_backward: accum is required"
BIG = 16 * 65535 + 1  # pixels: one tile more than a grid dimension holds

_ADAM_KEEP = []  # the arrays _adam_groups hands out stay alive for the whole module


def _adam_groups(*groups):
    """Host address of a gsr_adam_group array: one (numel, NULL member) pair per group, every other tensor a fake
    device address (the step reads the descriptors on the host and refuses a NULL tensor before any launch)."""
    from gaustudio_b200.optimizers import _AdamGroup
    arr = (_AdamGroup * len(groups))()
    for g, (numel, null) in zip(arr, groups):
        for i, f in enumerate(("param", "grad", "exp_avg", "exp_avg_sq")):
            setattr(g, f, None if f == null else (1 << 20) + 4096 * i)
        g.numel = numel
    _ADAM_KEEP.append(arr)
    return ctypes.addressof(arr)


NULL_GROUP = "gsr_adam_step: null tensor in a group"

# (entry point, fixed arguments, [(return value, gsr_last_error() or None, [argument overrides that trigger it]), ...]),
# the checks in the order they fire
CHECKS = [
    ("gsr_forward", {}, [
        (-1, POSITIVE, [{"P": 0}, {"width": 0}, {"height": -3}]),
        (-1, "gsr_forward: need shs or colors_precomp", [{"shs": None, "colors_precomp": None}]),
        (-1, "gsr_forward: need scales+rotations or cov3D_precomp",
         [{"cov3D_precomp": None, "scales": None}, {"cov3D_precomp": None, "rotations": None}]),
        (-1, "gsr_forward: rotations must be 16-byte aligned", [{"rotations": _Off(4)}]),
        (-1, SH_MISMATCH, [{"D": 4}, {"D": -1}, {"D": 1}]),
        (-1, TOO_LARGE, [{"width": BIG}, {"height": BIG}]),
        (-1, NO_SCRATCH, [{}, {"shs": None, "D": 3}, {"cov3D_precomp": None, "D": 1, "M": 4},
                          {"scales": None, "rotations": None}]),
    ]),
    ("gsr_forward_fused", {}, [
        (-1, POSITIVE, [{"P": 0}, {"width": -1}]),
        (-1, "gsr_forward_fused: need f_dc, f_rest, raw scales and rotations",
         [{"f_dc": None}, {"M": 4, "f_rest": None}, {"log_scales": None}, {"raw_rotations": None}, {"M": 0}]),
        (-1, "gsr_forward: rotations must be 16-byte aligned", [{"raw_rotations": _Off(8)}]),
        (-1, SH_MISMATCH, [{"D": 1}, {"D": 4, "M": 16}]),
        (-1, TOO_LARGE, [{"width": BIG}]),
        (-1, NO_SCRATCH, [{}, {"f_rest": None}, {"D": 3, "M": 16}]),
    ]),
    ("gsr_backward", {}, [
        (0, None, [{"P": 0}, {"P": -1}]),
        (-1, NO_STATE, [{"geom_buffer": None}, {"image_buffer": None}, {"binning_buffer": None, "R": 5}]),
        (-1, NO_BACKGROUND, [{"background": None}, {"background": None, "binning_buffer": None}]),
        (-1, NO_SCALES, [{"cov3D_precomp": None, "scales": None}, {"cov3D_precomp": None, "rotations": None}]),
        (-1, BWD_ALIGN, [{"rotations": _Off(4)}, {"scales": None, "rotations": None, "dL_drot": _Off(4)}]),
    ]),
    ("gsr_backward_fused", {}, [
        (0, None, [{"P": 0}]),
        (-1, NO_STATE, [{"geom_buffer": None}, {"image_buffer": None}, {"binning_buffer": None, "R": 1}]),
        (-1, NO_BACKGROUND, [{"background": None}]),
        (-1, NO_SCALES, [{"log_scales": None}, {"raw_rotations": None}]),
        (-1, BWD_ALIGN, [{"raw_rotations": _Off(4)}, {"dL_dcolor": None, "dL_dcov3D": None, "dL_draw_rot": _Off(12)}]),
    ]),
    ("gsr_debug_projection_backward", {"fused": 0}, [
        (-1, NO_ACCUM, [{"accum": None}]),
        (0, None, [{"P": 0}]),
        (-1, NO_STATE, [{"geom_buffer": None}]),
        (-1, NO_SCALES, [{"cov3D_precomp": None, "scales": None}, {"cov3D_precomp": None, "rotations": None}]),
        (-1, BWD_ALIGN, [{"rotations": _Off(4)}, {"scales": None, "rotations": None, "dL_dconic": _Off(4)}]),
    ]),
    ("gsr_debug_projection_backward", {"fused": 1}, [
        (-1, NO_ACCUM, [{"accum": None}]),
        (0, None, [{"P": 0}]),
        (-1, NO_STATE, [{"geom_buffer": None}]),
        (-1, NO_SCALES, [{"scales": None}, {"rotations": None}]),  # cov3D_precomp is ignored when fused
        (-1, BWD_ALIGN, [{"rotations": _Off(8)}]),
    ]),
    ("gsr_debug_accumulator", {}, [
        (-1, "gsr_debug_accumulator: geom_buffer and accum are required",
         [{"geom_buffer": None}, {"accum": None}, {"geom_buffer": None, "accum": None, "P": 0}]),
        (0, None, [{"P": 0}, {"P": -2}]),
    ]),
    ("gsr_mark_visible", {}, [
        (0, None, [{"P": 0}, {"P": -5}]),
        (-1, "gsr_mark_visible: null pointer", [{"means3D": None}, {"viewmatrix": None}, {"present": None}]),
    ]),
    ("gsr_depth2normal", {}, [
        (0, None, [{"width": 0}, {"height": -1}]),
        (-1, "gsr_depth2normal: null pointer", [{"depth": None}, {"out": None}, {"rot": None, "out": None}]),
    ]),
    ("gsr_depth2point", {}, [
        (0, None, [{"width": -1}, {"height": 0}]),
        (-1, "gsr_depth2point: null pointer", [{"depth": None}, {"out": None}, {"cam_to_world": None, "depth": None}]),
    ]),
    ("gsr_debug_export", {}, [
        (-1, "gsr_debug_export: missing state buffers",
         [{"geom_buffer": None}, {"image_buffer": None}, {"binning_buffer": None, "R": 5},
          {"geom_buffer": None, "P": 0, "point_list": None}]),
    ]),
    ("gsr_masked_bilateral", {}, [
        (0, None, [{"width": 0}, {"height": -1}]),
        (-1, "gsr_masked_bilateral: d must be odd, 1..15", [{"d": 0}, {"d": 4}, {"d": 17}, {"d": -1}]),
        (-1, "gsr_masked_bilateral: null pointer",
         [{"d": 5, p: None} for p in ("depth", "mask", "out_depth", "out_mask", "scratch")]),
    ]),
    ("gsr_extract_normals", {}, [
        (0, None, [{"width": 0}, {"height": 0}]),
        (-1, "gsr_extract_normals: null pointer",
         [{"filtered_depth": None}, {"fg_mask": None}, {"opacity": None}, {"median_depth": None}, {"rot": None},
          {"neg_world_normals": None}, {"valid": None}]),
    ]),
    ("gsr_normal_fusion_pass", {}, [
        (0, None, [{"n": 0}, {"n": -1}]),
        (-1, "gsr_normal_fusion_pass: null pointer",
         [{"n": 7, p: None} for p in ("ids", "normals", "confidences", "xyz", "sum_normals", "sum_weights")] +
         [{"n": 7, "P": 0}]),
    ]),
    ("gsr_normal_fusion_mean", {}, [
        (0, None, [{"P": 0}, {"P": -1}]),
    ]),
    ("gsr_knn_grid", {}, [
        (0, None, [{"n": 0}, {"n": -3, "k": 4}]),
        (-1, "gsr_knn_grid: null pointer",
         [{"n": 7, "k": 4, p: None} for p in ("points", "cell_start", "grid", "out_index", "out_dist")]),
        (-1, "gsr_knn_grid: k must be 1, 4, 8, 10 or 16", [{"n": 7, "k": 0}, {"n": 7, "k": 2}, {"n": 1, "k": 17}]),
    ]),
    ("gsr_adam_step", {}, [
        (0, None, [{"n_groups": 0}, {"n_groups": -1}]),
        (-1, "gsr_adam_step: 1..16 groups", [{"n_groups": 1, "groups": None}, {"n_groups": 17, "step": 1}]),
        (-1, "gsr_adam_step: step counts from 1", [{"n_groups": 1, "step": 0}, {"n_groups": 16, "step": -2}]),
        (-1, NULL_GROUP, [{"n_groups": 1, "step": 1, "groups": _adam_groups((4, m))}
                          for m in ("param", "grad", "exp_avg", "exp_avg_sq")] +
         [{"n_groups": 2, "step": 3, "groups": _adam_groups((0, "param"), (1, "exp_avg"))}]),
    ]),
]


@pytest.mark.parametrize("entry,fixed,checks", CHECKS,
                         ids=["forward", "forward_fused", "backward", "backward_fused", "debug_unfused", "debug_fused",
                              "debug_accumulator", "mark_visible", "depth2normal", "depth2point", "debug_export",
                              "masked_bilateral", "extract_normals", "normal_fusion_pass", "normal_fusion_mean",
                              "knn_grid", "adam_step"])
def test_argument_checks_fire_in_order_before_any_work(entry, fixed, checks):
    """Each argument check of the entry points listed returns its value and error text, alone and together with the
    triggers of every later check, so the order in which they fire is pinned too.  They all fire before the library
    touches memory or calls CUDA, which is why this runs without a GPU."""
    for k, (ret, err, variants) in enumerate(checks):
        later = {}
        for _, _, vs in reversed(checks[k + 1:]):
            later.update(vs[0])
        for v in variants:
            for over in (v, {**later, **v}):
                got = _call(entry, **fixed, **over)
                assert got == ret, (entry, fixed, over, got, _lib.last_error())
                if err is not None:
                    assert _lib.last_error() == err, (entry, fixed, over)


def test_misaligned_quaternions_are_refused_before_any_work():
    """The projection kernels read a Gaussian's quaternion (and write its gradient and dL_dconic) as one 16-byte vector.
    Each such pointer, at each offset that is not a multiple of 16 bytes, is refused with -1 and the alignment error,
    before the library touches memory or launches anything."""
    FWD_ALIGN = "gsr_forward: rotations must be 16-byte aligned"
    cases = [("gsr_forward", {}, ["rotations"], FWD_ALIGN),
             ("gsr_forward_fused", {}, ["raw_rotations"], FWD_ALIGN),
             ("gsr_backward", {}, ["rotations", "dL_drot", "dL_dconic"], BWD_ALIGN),
             ("gsr_backward_fused", {}, ["raw_rotations", "dL_draw_rot"], BWD_ALIGN),
             ("gsr_debug_projection_backward", {"fused": 0}, ["rotations", "dL_drot", "dL_dconic"], BWD_ALIGN),
             ("gsr_debug_projection_backward", {"fused": 1}, ["rotations", "dL_drot", "dL_dconic"], BWD_ALIGN)]
    for entry, fixed, names, err in cases:
        for name in names:
            for off in (4, 8, 12):
                assert _call(entry, **fixed, **{name: _Off(off)}) == -1, (entry, fixed, name, off)
                assert _lib.last_error() == err, (entry, fixed, name, off)


def test_no_oracle_import_in_product_path():
    """The product package must not reference oracle/ (a CPU fallback would void the parity claims)."""
    pkg = os.path.join(ROOT, "gaustudio_b200")
    for d, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(d, f)).read()
                assert "from oracle" not in txt and "import oracle" not in txt and "gsr_oracle" not in txt, f


def test_header_is_plain_c():
    """include/gsr.h is a C header: it must pass a C compiler on its own."""
    import subprocess
    subprocess.run(["gcc", "-x", "c", "-std=c99", "-Wall", "-Werror", "-fsyntax-only", os.path.join(ROOT, "include", "gsr.h")],
                   check=True)


def test_reference_side_binding_compiles_against_the_header():
    """integration/rasterize_points_gsr.cpp -- what the reference's rasterize_points.cu becomes on top of the C ABI
    (INTEGRATION.md section 3) -- type-checks against include/gsr.h, the torch headers and the CUDA runtime headers."""
    import subprocess
    import sysconfig
    from torch.utils import cpp_extension
    inc = [os.path.join(ROOT, "include"), sysconfig.get_paths()["include"], "/usr/local/cuda/include"]
    inc += cpp_extension.include_paths()
    cmd = ["g++", "-std=c++17", "-fsyntax-only", "-DTORCH_EXTENSION_NAME=_C", "-DTORCH_API_INCLUDE_EXTENSION_H"]
    for i in inc:
        cmd += ["-I", i]
    cmd.append(os.path.join(ROOT, "integration", "rasterize_points_gsr.cpp"))
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
