"""Builds libgsr_b200.so (hand-written sm_90a (H100) CUDA + the C ABI of include/gsr.h) in-tree with nvcc.

No fast-math: the reference extension is built without it ($RAST/setup.py:29), and the per-pair
thresholds of the compositing loop need the same precise expf / IEEE division.
"""
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SOURCES = ["gsr_api.cu", "gsr_preprocess.cu", "gsr_binning.cu", "gsr_render.cu", "gsr_extract.cu", "gsr_mesh.cu",
           "gsr_meshraster.cu", "gsr_surfel.cu", "gsr_mip.cu", "gsr_scaffold.cu", "gsr_densify.cu",
           "gsr_loss.cu", "gsr_adam.cu", "gsr_sap.cu", "gsr_clean.cu", "gsr_init.cu", "gsr_hull.cu"]
LIB = os.path.join(HERE, "libgsr_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "--expt-relaxed-constexpr",
         "--extended-lambda", "-Xcompiler", "-fPIC", "-Xptxas", "-v"]


def _stale(out):
    if not os.path.exists(out):
        return True
    t = os.path.getmtime(out)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h"))] + \
           [os.path.join(HERE, "..", "include", "gsr.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def _build(out, defines=(), force=False, verbose=False, log=None):
    """Compile SOURCES with FLAGS + defines (one nvcc per source, in parallel) and link them into `out`, whose soname is
    its file name.  Skipped unless forced or `out` is older than a csrc/ source or header or include/gsr.h.  The objects
    live in a temporary directory; the ptxas report goes to `log` (default: beside `out`)."""
    if not force and not _stale(out):
        return out
    os.makedirs(os.path.dirname(out), exist_ok=True)
    with tempfile.TemporaryDirectory() as tmp:
        objs = [os.path.join(tmp, s.replace(".cu", ".o")) for s in SOURCES]
        procs = [subprocess.Popen([NVCC, *FLAGS, *defines, "-c", os.path.join(CSRC, s), "-o", o],
                                  stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
                 for s, o in zip(SOURCES, objs)]
        outputs = [p.communicate()[0] for p in procs]
        text = "\n".join(f"==== {s}\n{o}" for s, o in zip(SOURCES, outputs))
        failed = [s for s, p in zip(SOURCES, procs) if p.returncode != 0]
        if failed:
            sys.stderr.write(text)
            raise RuntimeError(f"nvcc failed on {', '.join(failed)} ({os.path.basename(out)})")
        subprocess.check_call([NVCC, "-shared", "-Xlinker", f"-soname={os.path.basename(out)}", "-o", out, *objs,
                               "-lcudart", "-ldl"])
    with open(log or os.path.splitext(out)[0] + ".ptxas.log", "w") as f:
        f.write(text)
    if verbose:
        print(text)
    return out


def build_library(force=False, verbose=False):
    return _build(LIB, force=force, verbose=verbose, log=os.path.join(CSRC, "ptxas.log"))


STRESS_LIB = os.path.join(HERE, "libgsr_b200_stress.so")


def build_stress_variant(force=False):
    """Same sources with the compositing ring shrunk to ONE stage of 32 records (-DGSR_NSTAGE=1 -DGSR_RB=32): test
    infrastructure for tests/test_gpu_ring_stress.py (selected with GSR_LIB=<path>); never loaded by default."""
    return _build(STRESS_LIB, ["-DGSR_NSTAGE=1", "-DGSR_RB=32"], force=force)


if __name__ == "__main__":
    print(build_library(force="-f" in sys.argv, verbose=True))
