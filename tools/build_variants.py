"""Builds experiment variants of the library (extra -D flags) into gaustudio_b200/variants/libgsr_<name>.so; a variant is
selected at run time with GSR_LIB=<path> (see tools/block_size_ab.sh).  Test / measurement infrastructure only."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gaustudio_b200 import build as B  # noqa: E402

VARIANTS = {
    "pre64": ["-DGSR_PRE_THREADS=64"],
    "pre256": ["-DGSR_PRE_THREADS=256"],
    "exactexp": ["-DGSR_BWD_FASTEXP=0"],
    "bwd48": ["-DGSR_BWD_BOUND_EXTRA=32"],
    "tiny64": ["-DGSR_SORT_THREADS_TINY=64"],
    "tiny256": ["-DGSR_SORT_THREADS_TINY=256"],
    "tinycap1024": ["-DGSR_SORT_CAP_TINY=1024"],
    "tinycap4096": ["-DGSR_SORT_CAP_TINY=4096"],
    "tinycap4096_256": ["-DGSR_SORT_CAP_TINY=4096", "-DGSR_SORT_THREADS_TINY=256"],
    "tinycap1536": ["-DGSR_SORT_CAP_TINY=1536"],
    # experimental 8-CTA cluster tile scan compiled in (then GSR_SCAN_CLUSTER=1 selects it at run time; DESIGN.md 3.5)
    "cluster_scan": ["-DGSR_WITH_CLUSTER_SCAN=1"],
    "cluster_scan1024": ["-DGSR_WITH_CLUSTER_SCAN=1", "-DGSR_SCAN_CL_THREADS=1024"],
    # mesh rasterizer: faces with a clipped bounding box of up to N samples are drawn in place (default 64)
    "meshsmall16": ["-DGSR_MESH_SMALL_MAX=16"],
    "meshsmall256": ["-DGSR_MESH_SMALL_MAX=256"],
}


def build(names=None, force=False):
    for name, defs in VARIANTS.items():
        if not names or name in names:
            print(B._build(os.path.join(B.HERE, "variants", f"libgsr_{name}.so"), defs, force=force))


if __name__ == "__main__":
    build([a for a in sys.argv[1:] if a != "-f"], force="-f" in sys.argv)
