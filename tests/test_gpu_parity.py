"""-m gpu parity tests: the CUDA path (through the reference-shaped Python API -> ctypes -> C ABI) against
 (1) what the UNMODIFIED reference extension (oracle/_ref) computed on the same inputs on an H100, stored under
     tests/golden (tests/refgold.py: refgold_*.npz; ref_case_*.npz with the reference's sorted lists),
 (2) the CPU oracle.
Tolerances: BASELINE.json -- 1e-4 max-abs on images, 1e-3 relative on gradients.  Against the reference on the
same GPU the forward is expected to be BIT-EXACT (same arithmetic, same order), which is asserted."""
import os

import numpy as np
import pytest
import torch

import gpu_util as U
import refgold
import scenes
from oracle import ref_driver

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
FWD = ("color", "depth", "median", "opacity")


def _grad_keys(r):
    return sorted(k for k in r if k.startswith("g_"))


@pytest.mark.parametrize("case", "ABCD")
def test_matches_compiled_reference(case):
    s = scenes.scene(case)
    dev = torch.device("cuda")
    new = scenes.run_torch(s, U.new_rasterize, dev)
    ref = refgold.reference(f"case_{case}", lambda: scenes.run_torch(s, U.ref_rasterize, dev))
    for k in FWD + ("radii",):
        ref.assert_equal(k, new[k])
    assert _grad_keys(new) == _grad_keys(ref.names())
    for k in _grad_keys(new):
        a, b, scale = ref.pair(k, new[k])
        U.assert_grads_close(a, b, scale=scale, what=f"{case}:{k}")
    assert (new["radii"] > 0).any()


@pytest.mark.parametrize("case", "ABCD")
def test_matches_golden_fixture(case):
    f = os.path.join(GOLD, f"ref_case_{case}.npz")
    if not os.path.exists(f):
        pytest.skip("golden fixture missing")
    G = np.load(f)
    s = scenes.scene(case)
    U.assert_scene_matches_fixture(s, G)
    dev = torch.device("cuda")
    captured = {}

    def rast(rs, *a, **kw):
        res = U.new_rasterize(rs, *a, **kw)
        fn = res[0].grad_fn
        captured["R"], captured["bufs"] = fn.num_rendered, fn.saved_tensors[7:10]  # before backward frees them
        return res
    new = scenes.run_torch(s, rast, dev)
    R = captured["R"]
    assert R == int(G["ref_num_rendered"])
    assert np.array_equal(new["radii"], G["ref_radii"])
    from gaustudio_b200 import _C
    P = s["means3D"].shape[0]
    ex = _C.debug_export(P, s["W"], s["H"], R, *captured["bufs"])
    # global sort order: the reference's list minus (Gaussian, tile) pairs that cannot contribute (exact tile culling);
    # the tile boundaries of the fixture's list come from the pinned CPU oracle (its list equals the fixture's)
    from oracle.oracle import Oracle
    o = Oracle()
    o.forward(s["means3D"], s["opacities"], s["viewmatrix"], s["projmatrix"], s["campos"], s["tanfovx"], s["tanfovy"],
              s["W"], s["H"], s["D"], shs=s.get("shs"), colors_precomp=s.get("colors_precomp"), scales=s.get("scales"),
              rotations=s.get("rotations"), cov3D_precomp=s.get("cov3D_precomp"), scale_modifier=s["scale_modifier"])
    ob = o.binning()
    if np.array_equal(ob["point_list"], G["ref_point_list"]):  # (host libm may move a key by an ulp on another box)
        U.assert_binned_list_is_culled_reference_list(ex, G["ref_point_list"], ob["ranges"], s["W"], s["H"], P)
    for k in FWD:
        U.assert_images_close(new[k], G["ref_" + k], atol=1e-6, what=f"{case}:{k}")
    for k in _grad_keys(new):
        U.assert_grads_close(new[k], G["ref_" + k], what=f"{case}:{k}")


@pytest.mark.parametrize("case", "ABCD")
def test_matches_cpu_oracle(case):
    s = scenes.scene(case)
    new = scenes.run_torch(s, U.new_rasterize, torch.device("cuda"))
    orc = U.oracle_run(s)
    assert (new["radii"] != orc["radii"]).mean() < 1e-3
    for k in FWD:
        # 1e-4 max-abs; a hard-threshold flip (alpha<1/255, T<1e-4) moves a pixel by more, so a tiny budget
        U.assert_images_close(new[k], orc[k], atol=1e-4, outlier_frac=2e-3, what=f"{case}:{k}")
    for k in _grad_keys(new):
        a, b = new[k], orc[k]
        scale = np.abs(b).max()
        assert (np.abs(a - b) > 1e-3 * np.abs(b) + 2e-3 * scale).mean() < 2e-3, k


def test_sh_degrees_and_stride():
    """D < tensor degree: coefficients are read with stride M (quirk 13); every degree against the reference."""
    s = scenes.scene("A")
    for D in (0, 1, 2, 3):
        s["D"] = D
        new = scenes.run_torch(s, U.new_rasterize, torch.device("cuda"))
        ref = refgold.reference(f"sh_degree_{D}", lambda: scenes.run_torch(s, U.ref_rasterize, torch.device("cuda")))
        ref.assert_equal("color", new["color"], what=f"D={D} color")
        a, b, scale = ref.pair("g_shs", new["g_shs"])
        U.assert_grads_close(a, b, scale=scale, what=f"D={D} shs")
        assert (new["g_shs"][:, (D + 1) ** 2:, :] == 0).all()


def test_medium_scene_bit_exact_and_sorted():
    """cfg2-shaped scene (100k Gaussians, 800x800): forward bit-exact vs the reference; the sorted list is the
    reference's minus provably inert (Gaussian, tile) pairs, in the reference's order (checked on a fixed selection of
    tiles, the most crowded one included)."""
    import math
    from gaustudio_b200 import _C
    from gaustudio_b200.synthetic import build_config
    model, cams, c = build_config("cfg2", K=3)
    dev = torch.device("cuda")
    model.to(dev)
    e = torch.Tensor([])
    T = ((c["W"] + 15) // 16) * ((c["H"] + 15) // 16)
    for k, cam in enumerate(cams[:2]):
        cam.to(dev)
        with torch.no_grad():
            args = (torch.zeros(3, device=dev), model.get_attribute("xyz"), e, model.get_attribute("opacity"),
                    model.get_attribute("scale"), model.get_attribute("rot"), 1.0, e, cam.world_view_transform,
                    cam.full_proj_transform, math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5), c["H"], c["W"],
                    model.get_features.contiguous(), 3, cam.camera_center, False, False)
            n = _C.rasterize_gaussians(*args)

            def run_reference():
                r = ref_driver.module().rasterize_gaussians(*args)
                out = {"num_rendered": r[0], **{f"out{i}": r[i] for i in range(1, 6)}}
                out.update(U.reference_tile_segments(ref_driver.parse_binning(r[7], r[0]),
                                                     ref_driver.parse_image_ranges(r[8], c["W"] * c["H"], T), T, 1, 5, k))
                return out
            ref = refgold.reference(f"medium_view{k}", run_reference)
        R = ref.scalar("num_rendered")
        assert n[0] == R > 1_000_000
        for i in range(1, 6):
            ref.assert_equal(f"out{i}", n[i], what=f"output {i}")
        ex = _C.debug_export(c["P"], c["W"], c["H"], n[0], n[6], n[7], n[8])
        U.assert_binned_list_is_culled_reference_list(ex, ref.array("seg_list"), ref.array("seg_ranges"), c["W"], c["H"],
                                                      c["P"], tiles=ref.array("seg_tiles"))
        assert 0 < R - ex["num_binned"] < R // 2


def test_sparse_and_dense_projection_ctas_match_reference():
    """A scene whose projection CTAs are a mix of dense ones (everything visible) and sparse ones (most Gaussians
    behind the camera or far off screen, some off-screen centres whose splats still reach the image) stays
    bit-identical to the compiled reference; gradients within 1e-3."""
    s = dict(scenes.scene("D"))
    rng = np.random.RandomState(21)
    P = s["means3D"].shape[0]
    xyz, sc = s["means3D"].copy(), s["scales"].copy()
    far = np.arange(P) >= 1024
    far &= rng.rand(P) < 0.7                 # the first 1024 stay as they are: dense CTAs
    xyz[far] *= rng.uniform(3.0, 9.0, size=(int(far.sum()), 1)).astype(np.float32)   # behind the camera / off screen
    big = np.where(far)[0][:40]
    sc[big] = 1.5                            # off-screen centres whose splats still reach the image
    s["means3D"], s["scales"] = xyz, sc
    dev = torch.device("cuda")
    new = scenes.run_torch(s, U.new_rasterize, dev)
    ref = refgold.reference("sparse_dense", lambda: scenes.run_torch(s, U.ref_rasterize, dev))
    for k in FWD + ("radii",):
        ref.assert_equal(k, new[k])
    assert 0.2 < (new["radii"] > 0).mean() < 0.8
    assert _grad_keys(new) == _grad_keys(ref.names())
    for k in _grad_keys(new):
        a, b, scale = ref.pair(k, new[k])
        U.assert_grads_close(a, b, scale=scale, what=f"sparse:{k}")
