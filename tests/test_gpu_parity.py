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


# ---- images wider than one round of the tile scan (k_tile_scan: SCAN_TILES = 8192 tiles per round) -------------------
SCAN_ROUND = 8192


def pixel_scene(W, H, px, py, sigma_px, opacity, seed):
    """Gaussians centred on the given pixels with about sigma_px pixels of footprint, depths 1.5-4, SH degree 3, in the
    format of scenes.scene."""
    import math
    from test_gpu_compositing_f64 import _pix_to_u, _view_to_world
    rng = np.random.RandomState(seed)
    cam = scenes.camera(W, H, 50.0)
    tx, ty = math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5)
    P = len(px)
    z = rng.uniform(1.5, 4.0, P)
    u, v = _pix_to_u(np.asarray(px, np.float64), W, tx), _pix_to_u(np.asarray(py, np.float64), H, ty)
    fy = H / (2 * ty)
    s = (np.asarray(sigma_px, np.float64) * z / fy)[:, None] * np.exp(0.2 * rng.randn(P, 3))
    q = rng.randn(P, 4)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    return dict(W=W, H=H, D=3, means3D=f32(_view_to_world(cam, np.stack([u * z, v * z, z], 1))), scales=f32(s),
                rotations=f32(q), opacities=f32(np.broadcast_to(opacity, (P,))[:, None]),
                shs=f32(np.concatenate([rng.randn(P, 1, 3), 0.2 * rng.randn(P, 15, 3)], 1)),
                viewmatrix=cam.world_view_transform.numpy(), projmatrix=cam.full_proj_transform.numpy(),
                campos=cam.camera_center.numpy(), tanfovx=tx, tanfovy=ty)


def round_boundary_tiles(T):
    """The last and first tile of every round boundary the image has (8191, 8192, 16383, 16384, ...)."""
    return [t for b in range(SCAN_ROUND, T, SCAN_ROUND) for t in (b - 1, b)]


def wide_scene(key):
    W, H = {"3840x2160": (3840, 2160), "2561x1441": (2561, 1441), "strip_w": (16 * (SCAN_ROUND + 1), 16),
            "strip_h": (1, 16 * (SCAN_ROUND + 1)), "late_crowded": (3840, 2160)}[key]
    rng = np.random.RandomState(sum(map(ord, key)))
    gx, gy = (W + 15) // 16, (H + 15) // 16
    n = 3000
    # spread over the whole image, plus a few on each side of every round boundary and on the last tile
    tiles = np.concatenate([rng.randint(0, gx * gy, n), np.repeat(round_boundary_tiles(gx * gy) + [gx * gy - 1], 4)])
    px = (tiles % gx) * 16 + rng.uniform(0, 16, len(tiles))
    py = (tiles // gx) * 16 + rng.uniform(0, 16, len(tiles))
    px, py = np.minimum(px, W - 0.5), np.minimum(py, H - 0.5)
    sig = rng.uniform(1.0, 6.0, len(tiles))
    op = rng.uniform(0.1, 0.9, len(tiles))
    if key == "late_crowded":
        # dense clusters in tiles of the 2nd and the 3rd round: one for the 6k-12k sort tier, one for the > 12k tier
        for t, m in ((gx * 40 + 100, 8000), (gx * 80 + 100, 14000)):
            assert SCAN_ROUND <= t < gx * gy
            cx, cy = (t % gx) * 16 + 8, (t // gx) * 16 + 8
            px = np.concatenate([px, cx + rng.uniform(-5, 5, m)])
            py = np.concatenate([py, cy + rng.uniform(-5, 5, m)])
            sig = np.concatenate([sig, rng.uniform(1.0, 2.0, m)])
            op = np.concatenate([op, rng.uniform(0.02, 0.1, m)])
    return pixel_scene(W, H, px, py, sig, op, rng.randint(1 << 30))


def assert_ranges_are_one_scan(ranges, num_binned):
    """The tile ranges are what one exclusive scan over ALL tiles gives: non-empty ranges follow each other in tile
    order without gap or overlap from 0 to num_binned (the running total carried across the scan's rounds)."""
    rg = np.asarray(ranges.cpu()).astype(np.int64)
    n = rg[:, 1] - rg[:, 0]
    assert (n >= 0).all()
    assert not rg[n == 0].any(), "an empty tile has a non-zero range"
    live = rg[n > 0]
    assert live[0, 0] == 0, "the first non-empty range does not start at 0"
    assert (live[1:, 0] == live[:-1, 1]).all(), "ranges of consecutive non-empty tiles are not contiguous"
    assert live[-1, 1] == num_binned


@pytest.mark.parametrize("key", ["3840x2160", "2561x1441", "strip_w", "strip_h", "late_crowded"])
def test_multi_round_tile_scan_bit_exact_and_sorted(key):
    """Images of more than one tile-scan round: the forward is bit-exact against the reference, the sorted list is the
    reference's minus inert pairs on tiles of every round and at every round boundary, the ranges are one scan across
    all rounds, and the tile order of the launches changes nothing."""
    from gaustudio_b200 import _C
    s = wide_scene(key)
    W, H, P = s["W"], s["H"], s["means3D"].shape[0]
    gx, T = (W + 15) // 16, ((W + 15) // 16) * ((H + 15) // 16)
    assert T > SCAN_ROUND
    dev = torch.device("cuda")
    e = torch.Tensor([])
    d = lambda k: torch.as_tensor(s[k]).to(dev).contiguous()
    args = (torch.zeros(3, device=dev), d("means3D"), e, d("opacities"), d("scales"), d("rotations"), 1.0, e,
            d("viewmatrix"), d("projmatrix"), float(s["tanfovx"]), float(s["tanfovy"]), H, W, d("shs"), 3,
            d("campos"), False, False)
    n = _C.rasterize_gaussians(*args)
    rounds = [r * SCAN_ROUND for r in range((T + SCAN_ROUND - 1) // SCAN_ROUND)]

    def run_reference():
        r = ref_driver.module().rasterize_gaussians(*args)
        out = {"num_rendered": r[0], **{f"out{i}": r[i] for i in range(1, 6)}}
        rg = ref_driver.parse_image_ranges(r[8], W * H, T)
        cnt = (rg[:, 1] - rg[:, 0]).cpu().numpy()
        # two non-empty tiles of every round besides the boundaries and the most crowded tiles
        per_round = [t for r0 in rounds for t in np.nonzero(cnt[r0:r0 + SCAN_ROUND])[0][[0, -1]] + r0]
        out.update(U.reference_tile_segments(ref_driver.parse_binning(r[7], r[0]), rg, T, 3, 4, 0,
                                             extra=round_boundary_tiles(T) + [T - 1] + per_round))
        return out
    ref = refgold.reference(f"wide_{key}", run_reference)
    R = ref.scalar("num_rendered")
    assert n[0] == R
    for i in range(1, 6):
        ref.assert_equal(f"out{i}", n[i], what=f"{key}: output {i}")
    ex = _C.debug_export(P, W, H, n[0], n[6], n[7], n[8])
    seg_tiles = ref.array("seg_tiles")
    for t in round_boundary_tiles(T) + [T - 1]:
        assert t in seg_tiles
    assert all(((seg_tiles >= r0) & (seg_tiles < r0 + SCAN_ROUND)).any() for r0 in rounds)
    U.assert_binned_list_is_culled_reference_list(ex, ref.array("seg_list"), ref.array("seg_ranges"), W, H, P,
                                                  tiles=seg_tiles)
    assert ex["num_binned"] == _C.last_num_binned()
    assert_ranges_are_one_scan(ex["ranges"], ex["num_binned"])
    cnt = (ex["ranges"][:, 1] - ex["ranges"][:, 0]).cpu().numpy()
    # every round has binned tiles, and so do both sides of every boundary
    for r0 in rounds:
        assert cnt[r0:r0 + SCAN_ROUND].any(), f"round at tile {r0} is empty"
    for t in round_boundary_tiles(T):
        assert cnt[t] > 0, f"boundary tile {t} is empty"
    if key == "late_crowded":  # both crowded sort tiers draw tiles that a later round of the scan listed
        late = np.arange(T) >= SCAN_ROUND
        assert (late & (cnt > 6144) & (cnt <= 12288)).any() and (late & (cnt > 12288)).any(), sorted(cnt)[-4:]
    prev = _C.set_tile_order(0)
    try:
        for mode in (0, 2):
            _C.set_tile_order(mode)
            again = _C.rasterize_gaussians(*args)
            assert again[0] == n[0]
            for i in range(1, 6):
                assert torch.equal(again[i], n[i]), (key, mode, i)
    finally:
        _C.set_tile_order(prev)
