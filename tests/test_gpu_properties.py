"""Size-independent properties at BASELINE.json's full size (cfg 3: 1M Gaussians, 1920x1080)."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def big():
    from gaustudio_b200.synthetic import build_config
    model, cams, c = build_config("cfg3", K=8)
    dev = torch.device("cuda")
    model.to(dev)
    return model, [cm.to(dev) for cm in cams[:2]], c, dev


def _args(model, cam, c, dev):
    e = torch.Tensor([])
    with torch.no_grad():
        return (torch.zeros(3, device=dev), model.get_attribute("xyz"), e, model.get_attribute("opacity"),
                model.get_attribute("scale"), model.get_attribute("rot"), 1.0, e, cam.world_view_transform,
                cam.full_proj_transform, math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5), c["H"], c["W"],
                model.get_features.contiguous(), 3, cam.camera_center, False, False)


def test_full_size_binning_and_image_invariants(big):
    from gaustudio_b200 import _C
    model, cams, c, dev = big
    a = _args(model, cams[0], c, dev)
    R, color, depth, median, opacity, radii, gb, bb, ib = _C.rasterize_gaussians(*a)
    P, W, H = c["P"], c["W"], c["H"]
    ex = _C.debug_export(P, W, H, R, gb, bb, ib)
    # num_rendered keeps the reference's meaning (sum of the tile-rect areas); the binned list is shorter: pairs that
    # cannot reach alpha >= 1/255 anywhere in the tile are culled (their inertness is proven in test_gpu_parity /
    # test_gpu_fullsize against the reference's own list)
    assert R == int(ex["tiles_touched"].long().sum()) > 4_000_000
    Rb = ex["num_binned"]
    assert 0.4 * R < Rb < 0.95 * R
    rg = ex["ranges"].long()
    n = rg[:, 1] - rg[:, 0]
    assert int(n.sum()) == Rb
    nz = rg[n > 0]
    assert int(nz[0, 0]) == 0 and int(nz[-1, 1]) == Rb and torch.equal(nz[1:, 0], nz[:-1, 1])
    # per-tile order: ascending (depth bits, gaussian index) -- the reference's stable (tile|depth) sort
    ids = ex["point_list"].long()
    key = (ex["depths"].view(torch.int32).long()[ids] << 32) | ids
    tile_of = torch.repeat_interleave(torch.arange(rg.shape[0], device=dev), n)
    same = tile_of[1:] == tile_of[:-1]
    assert bool(((key[1:] > key[:-1]) | ~same).all())
    assert bool((torch.bincount(ids, minlength=P) <= ex["tiles_touched"].long()).all())
    assert torch.equal(opacity[0], 1 - ex["final_T"])
    assert float(opacity.min()) >= 0 and float(opacity.max()) <= 1 and bool(torch.isfinite(color).all())
    # n_contrib never exceeds the tile's list length
    Hp, Wp = (H + 15) // 16 * 16, (W + 15) // 16 * 16
    pad = torch.zeros(Hp, Wp, dtype=torch.int64, device=dev)
    pad[:H, :W] = ex["n_contrib"].long()
    assert bool((pad.view(Hp // 16, 16, Wp // 16, 16).amax(dim=(1, 3)).reshape(-1) <= n).all())
    # determinism of the forward (the level-1 scatter order is arbitrary, the result is not)
    again = _C.rasterize_gaussians(*a)
    for x, y in zip((color, depth, median, opacity, radii), again[1:6]):
        assert torch.equal(x, y)


def test_pipelined_equals_exact(big):
    from gaustudio_b200 import _C
    model, cams, c, dev = big
    exact = [_C.rasterize_gaussians(*_args(model, cam, c, dev)) for cam in cams]
    _C.set_pipelined(True)
    try:
        for rep in range(2):  # first call seeds the capacity, second is sync-free
            for cam, ex in zip(cams, exact):
                got = _C.rasterize_gaussians(*_args(model, cam, c, dev))
                for i in range(1, 6):
                    assert torch.equal(got[i], ex[i])
        _C.check_pipeline(wait=True)
    finally:
        _C.set_pipelined(False)


def test_backward_linearity_full_size(big):
    """grad is linear in the incoming pixel gradients: grad(2 dL) = 2 grad(dL), grad(dL1 + dL2) = sum."""
    from gaustudio_b200.rasterizer import GaussianRasterizationSettings, GaussianRasterizer
    model, cams, c, dev = big
    cam = cams[1]
    rs = GaussianRasterizationSettings(c["H"], c["W"], math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5),
                                       torch.zeros(3, device=dev), 1.0, cam.world_view_transform,
                                       cam.full_proj_transform, 3, cam.camera_center, False, False)
    g = torch.Generator().manual_seed(3)
    d1 = torch.randn(3, c["H"], c["W"], generator=g).to(dev)
    d2 = torch.randn(3, c["H"], c["W"], generator=g).to(dev)

    def grads(dl):
        with torch.no_grad():
            xyz = model.get_attribute("xyz").clone(); op = model.get_attribute("opacity").clone()
            sc = model.get_attribute("scale").clone(); rot = model.get_attribute("rot").clone()
            sh = model.get_features.clone()
        leaves = [t.requires_grad_(True) for t in (xyz, op, sc, rot, sh)]
        color, *_ = GaussianRasterizer(rs)(xyz, torch.zeros_like(xyz), op, shs=sh, scales=sc, rotations=rot)
        (color * dl).sum().backward()
        return [t.grad for t in leaves]
    ga, gb, g2, gs = grads(d1), grads(d2), grads(2 * d1), grads(d1 + d2)
    for a, b, two, s in zip(ga, gb, g2, gs):
        scale = float(a.abs().max()) + 1e-20
        assert float((two - 2 * a).abs().max()) <= 2e-4 * scale
        assert float((s - (a + b)).abs().max()) <= 2e-4 * (scale + float(b.abs().max()))
        assert bool(torch.isfinite(a).all())


def test_full_size_forward_bit_exact_vs_reference(big):
    """cfg 3 at full size (1M Gaussians, 1080p): all five forward outputs and num_rendered are bit-identical to the
    unmodified reference extension (golden data, tests/refgold.py); gradients of a random cotangent within 1e-3."""
    import refgold
    from oracle import ref_driver
    from gaustudio_b200 import _C
    from gaustudio_b200.rasterizer import GaussianRasterizationSettings, GaussianRasterizer
    model, cams, c, dev = big
    cam = cams[0]
    a = _args(model, cam, c, dev)
    new = _C.rasterize_gaussians(*a)
    rs = GaussianRasterizationSettings(c["H"], c["W"], math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5),
                                       torch.zeros(3, device=dev), 1.0, cam.world_view_transform,
                                       cam.full_proj_transform, 3, cam.camera_center, False, False)
    g = torch.Generator().manual_seed(11)
    wc = torch.randn(3, c["H"], c["W"], generator=g).to(dev); wd = torch.randn(1, c["H"], c["W"], generator=g).to(dev)

    def grads(fn):
        with torch.no_grad():
            leaves = [model.get_attribute("xyz").clone(), model.get_attribute("opacity").clone(),
                      model.get_attribute("scale").clone(), model.get_attribute("rot").clone(), model.get_features.clone()]
        xyz, op, sc, rot, sh = [t.requires_grad_(True) for t in leaves]
        color, radii, depth, median, opac = fn(rs, xyz, torch.zeros_like(xyz), op, shs=sh, scales=sc, rotations=rot)
        ((color * wc).sum() + (depth * wd).sum() + opac.sum()).backward()
        return [t.grad for t in (xyz, op, sc, rot, sh)]
    names = ("xyz", "opacity", "scale", "rot", "sh")

    def run_reference():
        r = ref_driver.module().rasterize_gaussians(*a)
        out = {"num_rendered": r[0], **{f"out{i}": r[i] for i in range(1, 6)}}
        del r
        out.update({"g_" + n: g for n, g in zip(names, grads(ref_driver.rasterize))})
        return out
    ref = refgold.reference("cfg3_full_size", run_reference)
    assert new[0] == ref.scalar("num_rendered")
    for i, name in zip(range(1, 6), ("color", "depth", "median", "opacity", "radii")):
        ref.assert_equal(f"out{i}", new[i], what=name)
    gn = grads(lambda rs_, *a_, **k: GaussianRasterizer(rs_)(*a_, **k))
    for name, x in zip(names, gn):
        x, y, scale = ref.pair("g_" + name, x)
        bad = (np.abs(x.astype(np.float64) - y) > 1e-3 * np.abs(y) + 1e-4 * scale).mean()
        assert float(bad) < 1e-5, (name, float(bad))
