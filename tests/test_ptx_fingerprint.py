"""The forward kernels are bit-identical to the reference only while nvcc contracts their plain C++ expressions into
the same mul / add / fma sequence (the reference is built with the default -fmad=true, and the parts that matter are
mirrored expression by expression).  A harmless-looking edit -- hoisting a load, reusing a product -- can flip one
mul+add pair into an fma and move a colour by an ulp; that only shows up in the `-m gpu` bit-exact tests.  This CPU test
pins the floating-point instruction sequence of the forward kernels' PTX to a committed fingerprint
(tests/golden/ptx_fp_fingerprint.json), so such a change is caught where there is no GPU.

After an INTENDED change of the forward arithmetic: run the GPU parity tests, then refresh the fingerprint with
`python tests/test_ptx_fingerprint.py --update`."""
import hashlib
import json
import os
import re
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "gaustudio_b200", "csrc")
GOLD = os.path.join(ROOT, "tests", "golden", "ptx_fp_fingerprint.json")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
# (source file, kernel-name fragment): the kernels whose outputs are compared bit for bit with the reference
KERNELS = [("gsr_preprocess.cu", "k_preprocess_fwd"), ("gsr_render.cu", "k_render_fwdILb0E")]
FP_OP = re.compile(r"^\s*(?:@%p\d+\s+)?((?:fma|mul|add|sub|div|rcp|sqrt|rsqrt|ex2|lg2|min|max|neg|abs|cvt)\.[a-z0-9.]*f32[a-z0-9.]*)\s")


def _fingerprints():
    out = {}
    for src, frag in KERNELS:
        ptx = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                              "--expt-relaxed-constexpr", "--extended-lambda", "-I", os.path.join(ROOT, "include"),
                              "-ptx", "-o", "/dev/stdout", os.path.join(CSRC, src)],
                             check=True, capture_output=True, text=True).stdout
        ops, inside = [], False
        for line in ptx.splitlines():
            if line.startswith((".visible .entry", ".entry", ".func", ".visible .func", ".weak .func")):
                inside = frag in line  # (a body runs to the next function header: inline-asm blocks hold braces at column 0)
            elif inside:
                m = FP_OP.match(line)
                if m:
                    ops.append(m.group(1))
        assert ops, f"{frag} not found in the PTX of {src}"
        out[frag] = {"n_ops": len(ops), "n_fma": sum(o.startswith("fma") for o in ops),
                     "sha256": hashlib.sha256("\n".join(ops).encode()).hexdigest()}
    return out


@pytest.mark.skipif(shutil.which(NVCC) is None and not os.path.exists(NVCC), reason="nvcc not available")
def test_forward_fp_sequence_matches_the_validated_one():
    assert os.path.exists(GOLD), "fingerprint missing: python tests/test_ptx_fingerprint.py --update"
    gold = json.load(open(GOLD))
    ver = subprocess.run([NVCC, "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
    if ver != gold["nvcc"]:
        pytest.skip(f"fingerprint was taken with another compiler ({gold['nvcc']}), this is {ver}")
    now = _fingerprints()
    for k in now:
        assert now[k] == gold["kernels"][k], (
            f"{k}: floating-point instruction sequence changed ({gold['kernels'][k]} -> {now[k]}); the forward may no "
            "longer be bit-identical to the reference.  Run the -m gpu parity tests, then refresh with --update")


if __name__ == "__main__":
    if "--update" in sys.argv:
        ver = subprocess.run([NVCC, "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
        json.dump({"nvcc": ver, "kernels": _fingerprints()}, open(GOLD, "w"), indent=1)
        print("wrote", GOLD)
    else:
        print(json.dumps(_fingerprints(), indent=1))
