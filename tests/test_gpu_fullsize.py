"""-m gpu parity at the FULL size of every BASELINE.json configuration a number is quoted on, in the mode it is
quoted in (VERDICT r1, next-round item 1):
  cfg 1  10k / 256x256, forward RGB           vs the CPU oracle and the compiled reference
  cfg 2  100k / 800x800, fwd+bwd              gradients vs the compiled reference
  cfg 3  1M / 1080p in bench.py's DEFAULT mode (fused activations + pipelined forward + one CUDA-graph replay per view)
         vs the compiled reference chained through the reference's torch activations
  cfg 5  5M / 1440x1080 forward only, D=3 and D=0 with M=16  vs the compiled reference (bit-exact, incl. sort order)
The compiled reference's results are golden data (tests/refgold.py).
Tolerances: BASELINE.json -- 1e-4 max-abs on images (bit-exact where the arithmetic is identical), 1e-3 relative on
gradients with a floor relative to the tensor's scale (the reference's own float atomics are order-dependent)."""
import math

import numpy as np
import pytest
import torch

import gpu_util as U
import refgold
from oracle import ref_driver, ref_torch_ops

pytestmark = pytest.mark.gpu
GRADS = ("xyz", "scale", "rot", "opacity", "f_dc", "f_rest")


def _rs(cls, cam, c, dev, D):
    return cls(c["H"], c["W"], math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5), torch.zeros(3, device=dev), 1.0,
               cam.world_view_transform, cam.full_proj_transform, D, cam.camera_center, False, False)


def _raw_args(model, cam, c, dev, D):
    e = torch.Tensor([])
    with torch.no_grad():
        return (torch.zeros(3, device=dev), model.get_attribute("xyz"), e, model.get_attribute("opacity"),
                model.get_attribute("scale"), model.get_attribute("rot"), 1.0, e, cam.world_view_transform,
                cam.full_proj_transform, math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5), c["H"], c["W"],
                model.get_features.contiguous(), D, cam.camera_center, False, False)


def _grad_bad_fraction(ref, key, x, rel=1e-3, floor=1e-4):
    """Fraction of the stored elements of gradient `key` where x is off the reference's by more than the tolerance."""
    a, b, scale = ref.pair(key, x)
    a, b = a.astype(np.float64), b.astype(np.float64)
    return float((np.abs(a - b) > rel * np.abs(b) + floor * scale).mean())


def _weights(c, dev, seed):
    g = torch.Generator().manual_seed(seed)
    H, W = c["H"], c["W"]
    return [torch.randn(s, H, W, generator=g).to(dev) for s in (3, 1, 1)]


def _weighted(out, w):
    return (out["render"] * w[0]).sum() + (out["rendered_depth"] * w[1]).sum() + (out["rendered_final_opacity"] * w[2]).sum()


def _reference_step(model, cam, c, dev, D, w):
    """The reference's op sequence: torch activations -> its CUDA extension -> loss -> backward (raw-attribute grads)."""
    for p in model.parameters_list():
        p.grad = None
    xyz, shs, opacity, scales, rotations = ref_torch_ops.gaussian_properties(model)
    color, radii, depth, median, opac = ref_driver.rasterize(_rs(ref_driver.RefSettings, cam, c, dev, D), xyz,
                                                             torch.zeros_like(xyz, requires_grad=True) + 0, opacity,
                                                             shs=shs, scales=scales, rotations=rotations)
    out = {"render": color, "rendered_depth": depth, "rendered_final_opacity": opac, "rendered_median": median,
           "radii": radii}
    _weighted(out, w).backward()
    res = {k: v.detach().clone() for k, v in out.items()}
    res.update({"g_" + n: p.grad.detach().clone() for n, p in zip(GRADS, model.parameters_list())})
    return res


def test_cfg1_real_size_forward_vs_oracle_and_reference():
    from gaustudio_b200 import _C
    from gaustudio_b200.synthetic import build_config
    from oracle.oracle import Oracle
    model, cams, c = build_config("cfg1")
    assert c["P"] == 10_000 and (c["W"], c["H"]) == (256, 256)
    dev = torch.device("cuda")
    cam = cams[0]
    o = Oracle()
    with torch.no_grad():
        orc = o.forward(model.get_attribute("xyz").numpy(), model.get_attribute("opacity").numpy(),
                        cam.world_view_transform.numpy(), cam.full_proj_transform.numpy(), cam.camera_center.numpy(),
                        math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5), 256, 256, 3, shs=model.get_features.numpy(),
                        scales=model.get_attribute("scale").numpy(), rotations=model.get_attribute("rot").numpy())
    model.to(dev); cam.to(dev)
    a = _raw_args(model, cam, c, dev, 3)
    new = _C.rasterize_gaussians(*a)

    def run_reference():
        r = ref_driver.module().rasterize_gaussians(*a)
        return {"num_rendered": r[0], **{f"out{i}": r[i] for i in range(1, 6)}}
    ref = refgold.reference("cfg1", run_reference)
    assert new[0] == ref.scalar("num_rendered") == orc["num_rendered"]
    for i in range(1, 6):
        ref.assert_equal(f"out{i}", new[i], what=f"output {i}")
    err = np.abs(new[1].cpu().numpy() - orc["color"])
    assert (err > 1e-4).mean() < 2e-3 and np.median(err) < 1e-6, err.max()
    assert (new[5].cpu().numpy() != orc["radii"]).mean() < 1e-3


def test_cfg2_full_size_gradients_vs_reference():
    from gaustudio_b200 import renderers
    from gaustudio_b200.synthetic import build_config
    model, cams, c = build_config("cfg2", K=4)
    assert c["P"] == 100_000 and (c["W"], c["H"]) == (800, 800)
    dev = torch.device("cuda")
    model.to(dev).requires_grad_(True)
    for k, cam in enumerate(cams[:2]):
        cam.to(dev)
        w = _weights(c, dev, 21 + k)
        ref = refgold.reference(f"cfg2_view{k}", lambda: _reference_step(model, cam, c, dev, 3, w))
        for fused in (False, True):
            for p in model.parameters_list():
                p.grad = None
            out = renderers.make({"name": "vanilla_renderer", "fused_activations": fused}).render(cam, model)
            _weighted(out, w).backward()
            if not fused:  # identical inputs -> identical forward
                ref.assert_equal("render", out["render"])
                ref.assert_equal("rendered_depth", out["rendered_depth"])
            for n, p in zip(GRADS, model.parameters_list()):
                bad = _grad_bad_fraction(ref, "g_" + n, p.grad)
                assert bad < 1e-5, (n, fused, bad)


def test_cfg3_bench_default_mode_matches_reference():
    """fused activations + pipelined (fixed-capacity) forward + CUDA-graph replay: the mode bench.py times."""
    from gaustudio_b200 import _C, renderers
    from gaustudio_b200.graphs import GraphedViewStep
    from gaustudio_b200.synthetic import build_config
    model, cams, c = build_config("cfg3", K=8)
    dev = torch.device("cuda")
    model.to(dev).requires_grad_(True)
    cams = [cm.to(dev) for cm in cams[:3]]
    w = _weights(c, dev, 5)
    r = renderers.make({"name": "vanilla_renderer", "fused_activations": True})
    before = _C.pipeline_state()
    step = GraphedViewStep(r, model, lambda out: _weighted(out, w), cams)
    assert _C.pipeline_state()["enabled"] == before["enabled"] and _C.pipeline_state()["fixed"] == before["fixed"]
    for k, cam in enumerate(cams[1:]):
        step(cam)                                         # one graph replay
        torch.cuda.synchronize()
        got = {k: step.out[k].detach().clone() for k in ("render", "rendered_depth", "rendered_final_opacity")}
        got_g = [g.detach().clone() for g in step.grads]
        ref = refgold.reference(f"cfg3_view{k}", lambda: _reference_step(model, cam, c, dev, 3, w))
        for key in got:
            a, b, _ = ref.pair(key, got[key])
            err = np.abs(a.astype(np.float64) - b)
            # fused exp / sigmoid / normalize round differently from the torch ops by ulps: a hard-threshold flip
            # (alpha < 1/255, T < 1e-4, tile rect) moves a pixel by more than 1e-4, hence a small outlier budget
            assert float((err > 1e-4).mean()) < 1e-3, (key, float(err.max()))
            assert float(np.median(err)) < 1e-6
        for n, x in zip(GRADS, got_g):
            bad = _grad_bad_fraction(ref, "g_" + n, x)
            assert bad < 1e-4, (n, bad)
    assert 0 < step.max_rendered() <= step.capacity


@pytest.mark.parametrize("D", [3, 0])
def test_cfg5_full_size_forward_bit_exact_vs_reference(D):
    """5M Gaussians, 1440x1080, the extraction-pass shape (forward only); D = 0 reads 12 of each 192-byte SH row
    (quirk 13).  All five outputs and num_rendered are identical to the reference's; the sorted list is the reference's
    minus provably inert (Gaussian, tile) pairs, in the reference's order (checked on a fixed selection of tiles, the
    most crowded one included)."""
    from gaustudio_b200 import _C
    from gaustudio_b200.synthetic import build_config
    model, cams, c = build_config("cfg5", K=8)
    assert c["P"] == 5_000_000 and (c["W"], c["H"]) == (1440, 1080)
    dev = torch.device("cuda")
    model.to(dev)
    cam = cams[1].to(dev)
    a = _raw_args(model, cam, c, dev, D)
    T = ((c["W"] + 15) // 16) * ((c["H"] + 15) // 16)
    with torch.no_grad():
        new = _C.rasterize_gaussians(*a)

        def run_reference():
            r = ref_driver.module().rasterize_gaussians(*a)
            out = {"num_rendered": r[0], **{f"out{i}": r[i] for i in range(1, 6)}}
            out.update(U.reference_tile_segments(ref_driver.parse_binning(r[7], r[0]),
                                                 ref_driver.parse_image_ranges(r[8], c["W"] * c["H"], T), T, 1, 3, D))
            return out
        ref = refgold.reference(f"cfg5_D{D}", run_reference)
    R = ref.scalar("num_rendered")
    assert new[0] == R > 10_000_000
    for i, name in zip(range(1, 6), ("color", "depth", "median", "opacity", "radii")):
        ref.assert_equal(f"out{i}", new[i], what=name)
    ex = _C.debug_export(c["P"], c["W"], c["H"], new[0], new[6], new[7], new[8])
    U.assert_binned_list_is_culled_reference_list(ex, ref.array("seg_list"), ref.array("seg_ranges"), c["W"], c["H"],
                                                  c["P"], tiles=ref.array("seg_tiles"))
    assert 0 < R - ex["num_binned"] < R
    n = (ex["ranges"][:, 1] - ex["ranges"][:, 0]).long()
    assert int(n.max()) > 4096, int(n.max())  # the crowded-tile sort tier is exercised (larger tiers: test_gpu_api)
    del new, ex
    torch.cuda.empty_cache()
