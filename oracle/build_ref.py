"""Build the UNMODIFIED reference rasterizer (CUDA) as a GPU-side parity oracle.

TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is imported by the product
path (gaustudio_b200/); only tests/, __graft_entry__.smoke() and bench.py's
reference / cpu_baseline legs may use it.

Compiles, from the sources *where they lie* under /root/reference (nothing is
copied into this repo), the reference's pybind11 extension

    $RAST/cuda_rasterizer/{rasterizer_impl,forward,backward}.cu
    $RAST/rasterize_points.cu, $RAST/ext.cpp          (setup.py:18-29)

for sm_90a into  oracle/_ref/_refC.so  (git-ignored, never committed).  The reference's own build system (setup.py / CMake) is NOT run;
this is the same five translation units + `-I third_party/glm` that
`$RAST/setup.py:24-29` lists, handed to torch.utils.cpp_extension.load.

Usage:  python oracle/build_ref.py
"""
import os
import shutil
import sys

RAST = "/root/reference/submodules/gaustudio-diff-gaussian-rasterization"
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
NAME = "_refC"


def so_path():
    return os.path.join(OUT, NAME + ".so")


def build(verbose=False):
    if not os.path.isdir(RAST):
        return None  # GPU box: only the prebuilt .so is available
    if os.path.exists(so_path()):
        return so_path()
    os.makedirs(OUT, exist_ok=True)
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    os.environ.setdefault("MAX_JOBS", "8")
    from torch.utils import cpp_extension

    srcs = [
        f"{RAST}/cuda_rasterizer/rasterizer_impl.cu",
        f"{RAST}/cuda_rasterizer/forward.cu",
        f"{RAST}/cuda_rasterizer/backward.cu",
        f"{RAST}/rasterize_points.cu",
        f"{RAST}/ext.cpp",
    ]
    bdir = os.path.join(OUT, "build")
    os.makedirs(bdir, exist_ok=True)
    cpp_extension.load(
        name=NAME,
        sources=srcs,
        extra_include_paths=[f"{RAST}/third_party/glm", RAST],
        extra_cuda_cflags=["-gencode=arch=compute_90a,code=sm_90a", "-lineinfo"],
        build_directory=bdir,
        verbose=verbose,
        is_python_module=True,
    )
    shutil.copy(os.path.join(bdir, NAME + ".so"), so_path())
    shutil.rmtree(bdir, ignore_errors=True)
    return so_path()


if __name__ == "__main__":
    p = build(verbose=True)
    print("reference oracle:", p)
    sys.exit(0 if p else 1)
