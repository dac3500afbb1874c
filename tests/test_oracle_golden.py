"""Pins the CPU oracle: oracle vs the golden tensors the unmodified reference CUDA extension produced on a
GPU (tests/golden/ref_case_*.npz, generator tests/golden/make_golden_ref.py).  Runs without a GPU."""
import os

import numpy as np
import pytest

import gpu_util as U
import scenes

GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.mark.parametrize("case", "ABCD")
def test_oracle_reproduces_reference_outputs(case):
    f = os.path.join(GOLD, f"ref_case_{case}.npz")
    if not os.path.exists(f):
        pytest.skip("golden fixture missing (generate on the GPU box)")
    G = np.load(f)
    s = scenes.scene(case)
    U.assert_scene_matches_fixture(s, G)
    orc = U.oracle_run(s)
    assert abs(orc["num_rendered"] - int(G["ref_num_rendered"])) <= 2
    assert (orc["radii"] != G["ref_radii"]).mean() < 1e-3
    for k in ("color", "depth", "median", "opacity"):
        U.assert_images_close(orc[k], G["ref_" + k], atol=1e-4, outlier_frac=2e-3, what=f"{case}:{k}")
    for k in sorted(x for x in orc if x.startswith("g_")):
        a, b = orc[k], G["ref_" + k]
        scale = np.abs(b).max()
        assert (np.abs(a - b) > 1e-3 * np.abs(b) + 2e-3 * scale).mean() < 2e-3, k
