"""Generates tests/golden/ref_case_*.npz by running the UNMODIFIED reference CUDA extension
(oracle/_ref/_refC.so, built by oracle/build_ref.py from the reference sources) on an H100:

    python tests/golden/make_golden_ref.py [OUT_DIR]     # writes OUT_DIR/ref_case_*.npz (default: tests/golden)

Each file holds the digests of the input arrays and the scalar inputs (tests/gpu_util.py::assert_scene_matches_fixture),
the reference's 5 outputs, num_rendered, its sorted point_list and its 8 gradients.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import ref_driver  # noqa: E402
import gpu_util  # noqa: E402
import scenes  # noqa: E402

out_dir = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden")
os.makedirs(out_dir, exist_ok=True)
dev = torch.device("cuda")
for case in "ABCD":
    s = scenes.scene(case)
    captured = {}
    def rasterize(rs, *a, **k):
        res = ref_driver.rasterize(rs, *a, **k)
        fn = res[0].grad_fn
        captured["binning"], captured["R"] = fn.saved_tensors[8], fn.num_rendered  # before backward frees them
        return res
    r = scenes.run_torch(s, rasterize, dev)
    binning, R = captured["binning"], captured["R"]
    r["num_rendered"] = np.int64(R)
    r["point_list"] = ref_driver.parse_binning(binning, R).cpu().numpy()
    save = {("insha_" + k): np.asarray(gpu_util.array_digest(v)) for k, v in s.items() if isinstance(v, np.ndarray)}
    save.update({("in_" + k): np.asarray(v) for k, v in s.items() if isinstance(v, (int, float))})
    save.update({("ref_" + k): v for k, v in r.items()})
    np.savez_compressed(os.path.join(out_dir, f"ref_case_{case}.npz"), **save)
    print(case, "R", R, "visible", int((r["radii"] > 0).sum()), {k: v.shape for k, v in r.items() if hasattr(v, "shape")})
