"""Builds integration/rasterize_points_gsr.cpp -- the reference's pybind module on top of the C ABI of libgsr_b200.so --
into integration/_gsr_refbind.so (git-ignored).  It exposes the same three
functions as the reference's `_C` (ext.cpp:15-19), so `tests/test_gpu_binding.py` can run the reference's own Python
autograd wrapper shape over it and compare with the ctypes path.  Plain C++ (no CUDA in this translation unit)."""
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
NAME = "_gsr_refbind"


def so_path():
    return os.path.join(HERE, NAME + ".so")


def build(verbose=False, force=False):
    src = os.path.join(HERE, "rasterize_points_gsr.cpp")
    deps = [src, os.path.join(ROOT, "include", "gsr.h")]
    if not force and os.path.exists(so_path()) and all(os.path.getmtime(so_path()) >= os.path.getmtime(d) for d in deps):
        return so_path()
    from torch.utils import cpp_extension
    libdir = os.path.join(ROOT, "gaustudio_b200")
    bdir = os.path.join(HERE, "build")
    os.makedirs(bdir, exist_ok=True)
    # no rpath: libgsr_b200.so is mapped first (here and in `load()`), the module's NEEDED entry then resolves by soname
    import ctypes
    ctypes.CDLL(os.path.join(libdir, "libgsr_b200.so"), mode=ctypes.RTLD_GLOBAL)
    cpp_extension.load(name=NAME, sources=[src], extra_include_paths=[os.path.join(ROOT, "include")],
                       extra_ldflags=[f"-L{libdir}", "-lgsr_b200"], with_cuda=True, build_directory=bdir,
                       verbose=verbose, is_python_module=True)
    shutil.copy(os.path.join(bdir, NAME + ".so"), so_path())
    shutil.rmtree(bdir, ignore_errors=True)
    return so_path()


def load():
    """Import the built module (None if it was never built)."""
    if not os.path.exists(so_path()):
        return None
    import ctypes
    import importlib.util
    import torch  # noqa: F401  (libtorch / libc10 must be mapped first)
    ctypes.CDLL(os.path.join(ROOT, "gaustudio_b200", "libgsr_b200.so"), mode=ctypes.RTLD_GLOBAL)
    spec = importlib.util.spec_from_file_location(NAME, so_path())
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    print(build(verbose=True, force="-f" in sys.argv))
