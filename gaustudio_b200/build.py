"""Builds libgsr_b200.so (hand-written sm_90a (H100) CUDA + the C ABI of include/gsr.h) in-tree with nvcc.

No fast-math: the reference extension is built without it ($RAST/setup.py:29), and the per-pair
thresholds of the compositing loop need the same precise expf / IEEE division.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SOURCES = ["gsr_api.cu", "gsr_preprocess.cu", "gsr_binning.cu", "gsr_render.cu", "gsr_extract.cu", "gsr_mesh.cu",
           "gsr_meshraster.cu", "gsr_surfel.cu", "gsr_mip.cu", "gsr_scaffold.cu", "gsr_densify.cu",
           "gsr_loss.cu", "gsr_adam.cu"]
LIB = os.path.join(HERE, "libgsr_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "--expt-relaxed-constexpr",
         "--extended-lambda", "-Xcompiler", "-fPIC", "-Xptxas", "-v"]


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h"))] + \
           [os.path.join(HERE, "..", "include", "gsr.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build_library(force=False, verbose=False):
    if not force and not _stale():
        return LIB
    objs = []
    procs = []
    for s in SOURCES:
        o = os.path.join(CSRC, s.replace(".cu", ".o"))
        objs.append(o)
        cmd = [NVCC, *FLAGS, "-c", os.path.join(CSRC, s), "-o", o]
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    for s, p in procs:
        out, _ = p.communicate()
        log.append(f"==== {s}\n{out}")
        if p.returncode != 0:
            sys.stderr.write("\n".join(log))
            raise RuntimeError(f"nvcc failed on {s}")
    subprocess.check_call([NVCC, "-shared", "-Xlinker", "-soname=libgsr_b200.so", "-o", LIB, *objs, "-lcudart", "-ldl"])
    text = "\n".join(log)
    with open(os.path.join(CSRC, "ptxas.log"), "w") as f:
        f.write(text)
    if verbose:
        print(text)
    return LIB


STRESS_LIB = os.path.join(HERE, "libgsr_b200_stress.so")


def build_stress_variant(force=False):
    """Same sources with the compositing ring shrunk to ONE stage of 32 records (-DGSR_NSTAGE=1 -DGSR_RB=32): test
    infrastructure for tests/test_gpu_ring_stress.py (selected with GSR_LIB=<path>); never loaded by default."""
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh"))]
    if not force and os.path.exists(STRESS_LIB) and all(os.path.getmtime(STRESS_LIB) >= os.path.getmtime(d) for d in deps):
        return STRESS_LIB
    objs, procs = [], []
    for s in SOURCES:
        o = os.path.join(CSRC, s.replace(".cu", ".stress.o"))
        objs.append(o)
        flags = [f for f in FLAGS if f not in ("-Xptxas", "-v")] + ["-DGSR_NSTAGE=1", "-DGSR_RB=32"]
        procs.append((s, subprocess.Popen([NVCC, *flags, "-c", os.path.join(CSRC, s), "-o", o], stdout=subprocess.PIPE,
                                          stderr=subprocess.STDOUT, text=True)))
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError(f"nvcc failed on {s} (stress variant)")
    subprocess.check_call([NVCC, "-shared", "-Xlinker", "-soname=libgsr_b200_stress.so", "-o", STRESS_LIB, *objs, "-lcudart", "-ldl"])
    for o in objs:
        os.remove(o)
    return STRESS_LIB


if __name__ == "__main__":
    print(build_library(force="-f" in sys.argv, verbose=True))
