"""-m gpu: the Scaffold-GS path -- anchor visibility against the Mip forward's radii, the CUDA decoding against the float64
restatement of the reference (tests/scaffold_ref64.py), and the scaffold_renderer end to end."""
import math

import numpy as np
import pytest
import torch

import scaffold_ref64 as SR
import scaffold_scenes as SS
from gpu_util import assert_grads_close

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")


def _mip_rasterizer(cam, k, mod):
    from gaustudio_b200.mip_rasterizer import GaussianRasterizationSettings, GaussianRasterizer
    rs = GaussianRasterizationSettings(
        image_height=int(cam.image_height), image_width=int(cam.image_width), tanfovx=math.tan(cam.FoVx * 0.5),
        tanfovy=math.tan(cam.FoVy * 0.5), kernel_size=k, bg=torch.zeros(3), scale_modifier=mod,
        viewmatrix=cam.world_view_transform, projmatrix=cam.full_proj_transform, sh_degree=1,
        campos=cam.camera_center, prefiltered=False, debug=False)
    return GaussianRasterizer(rs)


def _cov3d(s, q):
    r, x, y, z = torch.nn.functional.normalize(q).unbind(1)
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                     2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                     2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)
    L = R * s[:, None, :]
    S = L @ L.transpose(1, 2)
    return torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], 1).contiguous()


@pytest.mark.parametrize("pre", [False, True], ids=["scales", "precomp"])
@pytest.mark.parametrize("mod", [1.0, 0.7])
@pytest.mark.parametrize("k", [0.0, 0.1, 0.3])
def test_visible_filter_radii_equal_the_mip_forward_radii(k, mod, pre):
    m = SS.model(20000, 4, F=8, seed=int(10 * k) + int(10 * mod), device="cuda")
    cam = SS.camera(320, 240, device="cuda")
    xyz = m.get_attribute("anchor")
    scales, rots = m.get_attribute("scale")[:, :3].contiguous(), m.get_attribute("rot")
    with torch.no_grad():  # a spread of sizes, down to degenerate ones
        scales = scales * torch.exp(2.0 * torch.randn(scales.shape, generator=torch.Generator().manual_seed(1))).to(DEV)
    r = _mip_rasterizer(cam, k, mod)
    geo = dict(cov3D_precomp=_cov3d(mod * scales, rots)) if pre else dict(scales=scales, rotations=rots)
    # with precomputed covariances the modifier is not applied: the forward ignores it as well
    radii = r.visible_filter(xyz, **geo)
    n = xyz.shape[0]
    _, fw_radii, *_ = r(xyz, torch.zeros_like(xyz), torch.full((n, 1), 0.5, device=DEV),
                        colors_precomp=torch.rand(n, 3, device=DEV), **geo)
    assert radii.dtype == torch.int32 and torch.equal(radii, fw_radii)
    vis = int((radii > 0).sum())
    assert 0.5 * n < vis < n, vis
    assert int((radii == 0).sum()) >= n // 25  # behind the camera (most off-screen ones too, unless very large)


def _gpu(case):
    return {n: t.to(DEV) for n, t in case.items()}


def _row_check(a, b, rtol, atol, what):
    """||a_i - b_i|| <= rtol ||b_i|| + atol max_j ||b_j|| per row: the floor covers rows that are sums or differences
    of larger terms (an anchor's gradient summed over its offsets, an xyz near the origin)."""
    a, b = a.double().reshape(a.shape[0], -1), b.double().reshape(b.shape[0], -1)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    err = (a - b).norm(dim=1)
    bn = b.norm(dim=1)
    bound = rtol * bn + atol * (float(bn.max()) if bn.numel() else 0.0) + 1e-30
    bad = err > bound
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} rows over, worst {float((err / (b.norm(dim=1) + 1e-30)).max()):.3g}"


def _decode(c):
    from gaustudio_b200 import _C
    base, M = _C.scaffold_count(c["opacity"])
    out = _C.scaffold_decode(c["vis"], base, M, c["anchor"], c["offset"], c["scaling"], c["opacity"], c["color"],
                             c["cov"])
    return base, M, out


@pytest.mark.parametrize("k", [1, 10, 32])
def test_decode_forward_against_the_f64_restatement(k):
    c = _gpu(SS.decode_case(5000, k, 100 + k))
    base, M, out = _decode(c)
    ref = SR.decode(**{n: (t.double() if t.is_floating_point() else t) for n, t in c.items()})
    assert M == ref[0].shape[0] and 0 < M < c["opacity"].numel()
    assert out[4].data_ptr() % 16 == 0 and out[2].shape == (M, 1)
    assert torch.equal(out[2], ref[2].float())  # opacities are copied: same rows in the same order
    for name, a, b in zip(("xyz", "rgb", "opacity", "scales", "rotations"), out, ref[:5]):
        _row_check(a, b, 1e-6, 1e-7, name)
    # the per-anchor prefix
    kept = (c["opacity"] > 0).sum(1)
    assert torch.equal(base.long(), torch.cat([torch.zeros(1, device=DEV, dtype=torch.long), kept.cumsum(0)]))


def test_decode_with_nothing_kept_or_nothing_visible():
    from gaustudio_b200 import _C
    c = _gpu(SS.decode_case(400, 10, 3))
    c["opacity"] = -c["opacity"].abs()
    base, M, out = _decode(c)
    assert M == 0 and all(t.shape[0] == 0 for t in out)
    g = _C.scaffold_decode_backward(c["vis"], base, M, c["offset"], c["scaling"], c["opacity"], c["cov"], [None] * 5)
    assert all(not bool(t.any()) for t in g)
    c = _gpu(SS.decode_case(400, 10, 3, frac=0.0))
    assert c["vis"].numel() == 0
    base, M, out = _decode(c)
    assert M == 0 and base.shape == (1,) and int(base[0]) == 0
    g = _C.scaffold_decode_backward(c["vis"], base, M, c["offset"], c["scaling"], c["opacity"], c["cov"], [None] * 5)
    assert [tuple(t.shape) for t in g] == [(400, 3), (400, 10, 3), (400, 6), (0, 10), (0, 30), (0, 70)]
    assert all(not bool(t.any()) for t in g)


@pytest.mark.parametrize("k", [1, 10, 32])
def test_decode_backward_against_f64_autograd(k):
    from gaustudio_b200 import _C
    c = _gpu(SS.decode_case(3000, k, 200 + k))
    base, M, out = _decode(c)
    g = torch.Generator().manual_seed(k)
    ups = [torch.randn(t.shape, generator=g).to(DEV) for t in out]
    got = _C.scaffold_decode_backward(c["vis"], base, M, c["offset"], c["scaling"], c["opacity"], c["cov"], ups)
    again = _C.scaffold_decode_backward(c["vis"], base, M, c["offset"], c["scaling"], c["opacity"], c["cov"], ups)
    for a, b in zip(got, again):
        assert torch.equal(a, b), "two runs differ"
    names = ("anchor", "offset", "scaling", "opacity", "color", "cov")
    leaves = {n: c[n].double().requires_grad_(True) for n in names}
    ref = SR.decode(c["vis"], **leaves)
    torch.autograd.backward(ref[:5], [u.double() for u in ups])
    N = c["anchor"].shape[0]
    invisible = torch.ones(N, dtype=torch.bool, device=DEV)
    invisible[c["vis"]] = False
    dropped = ~(c["opacity"] > 0)
    for name, a in zip(names, got):
        b = leaves[name].grad
        assert a.shape == b.shape, name
        if name in ("anchor", "offset", "scaling"):
            assert not bool(a[invisible].any()), f"{name}: non-zero on an invisible anchor"
            if name == "offset":
                assert not bool(a[c["vis"]][dropped].any()), "offset: non-zero on a dropped offset"
            rows = ~invisible
            if name == "offset":
                a, b = a[c["vis"]][~dropped], b[c["vis"]][~dropped]
            else:
                a, b = a[rows], b[rows]
        else:
            w = {"opacity": 1, "color": 3, "cov": 7}[name]
            a3, b3 = a.view(-1, k, w), b.view(-1, k, w)
            assert not bool(a3[dropped].any()), f"{name}: non-zero on a dropped offset"
            a, b = a3[~dropped], b3[~dropped]
        _row_check(a, b, 1e-5, 1e-6, name)


# ---- end to end -------------------------------------------------------------------------------------------------
def _torch_render(r, cam, m):
    """The Mip rasterizer fed the fp32 torch restatement of the reference's decoding (same visibility and MLPs)."""
    from gaustudio_b200 import scaffold
    from gaustudio_b200.renderers.base import pack_result
    visible = r.prefilter_voxel(cam, m)
    vis = visible.nonzero().flatten()
    o, c, s = scaffold.mlp_outputs(m, vis, cam.camera_center)
    xyz, rgb, op, sc, rot, _ = SR.decode(vis, m.get_attribute("anchor"), m.get_attribute("offset"),
                                         m.get_attribute("scale"), o, c, s)
    (img, radii, depth, med, fo), ss = r.rasterize(cam, m, (xyz, None, rgb, op, sc, rot.contiguous(), None))
    return pack_result(img, radii, depth, med, fo, ss)


def _params(m):
    p = {"anchor_feat": m._anchor_feat, "offset": m._offset, "scale": m._scale}
    for name, mlp in m.mlps().items():
        for pn, t in mlp.named_parameters():
            p[f"{name}.{pn}"] = t
    return p


@pytest.mark.parametrize("bank", [False, True], ids=["plain", "feature_bank"])
def test_renderer_matches_the_torch_decoding_end_to_end(bank):
    from gaustudio_b200 import renderers
    r = renderers.make({"name": "scaffold_renderer", "kernel_size": 0.1})
    m = SS.model(3000, 10, F=32, seed=11, use_feat_bank=bank, device="cuda").requires_grad_(True)
    cam = SS.camera(device="cuda")
    w = torch.randn(3, SS.H, SS.W, generator=torch.Generator().manual_seed(2)).to(DEV)
    outs, grads = [], []
    for fn in (lambda: r.render(cam, m), lambda: _torch_render(r, cam, m)):
        out = fn()
        ((out["render"] * w).sum() + out["rendered_depth"].sum()).backward()
        p = _params(m)
        grads.append({n: t.grad.clone() for n, t in p.items()})
        for t in p.values():
            t.grad = None
        outs.append(out)
    a, b = outs
    assert torch.equal(a["radii"], b["radii"])
    assert int((a["radii"] > 0).sum()) > 5000
    for key in ("render", "rendered_depth", "rendered_final_opacity"):
        assert float((a[key] - b[key]).detach().abs().max()) <= 1e-4, key
    assert set(a) >= {"visible_mask", "selection_mask", "neural_opacity", "scaling"}
    Nv = int(a["visible_mask"].sum())
    assert a["selection_mask"].shape == (Nv * 10,) and a["neural_opacity"].shape == (Nv * 10, 1)
    assert a["scaling"].shape == (int(a["selection_mask"].sum()), 3) == (a["radii"].shape[0], 3)
    for n in grads[1]:
        assert_grads_close(grads[0][n].cpu(), grads[1][n].cpu(), what=n)


def test_outputs_do_not_depend_on_an_earlier_scene():
    from gaustudio_b200 import renderers
    r = renderers.make("scaffold_renderer")
    cam = SS.camera(device="cuda")
    A = SS.model(4000, 10, F=16, seed=21, device="cuda")
    B = SS.model(6000, 10, F=16, seed=22, device="cuda")
    keys = ("render", "rendered_depth", "rendered_median_depth", "rendered_median_id", "rendered_final_opacity", "radii",
            "visible_mask", "selection_mask", "neural_opacity", "scaling")
    with torch.no_grad():
        a1 = r.render(cam, A)
        r.render(cam, B)
        a2 = r.render(cam, A)
    for key in keys:
        assert torch.equal(a1[key], a2[key]), key


def _fit(r, cams, targets, m, lrs, steps=200):
    opt = torch.optim.Adam([{"params": [m._anchor_feat], "lr": lrs[0]}, {"params": [m._offset], "lr": lrs[1]},
                            {"params": [m._scale], "lr": lrs[2]},
                            {"params": [p for mlp in m.mlps().values() for p in mlp.parameters()], "lr": lrs[3]}])
    losses = []
    for it in range(steps):
        loss = (r.render(cams[it % len(cams)], m)["render"] - targets[it % len(cams)]).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    return np.mean(losses[:8]), np.mean(losses[-8:])


def _perturbed(target, seed):
    """The target with its features and the MLPs' output layers perturbed by noise of another seed (the colour layer
    most); offsets and scales start at the target's and are trained along."""
    import copy
    m = copy.deepcopy(target)
    g = torch.Generator(device="cuda").manual_seed(seed)
    noise = lambda t, s: t + s * torch.randn(t.shape, generator=g, device="cuda")
    with torch.no_grad():
        m._anchor_feat = noise(m._anchor_feat, 1.5)
        for name, mlp in m.mlps().items():
            mlp[2].weight.copy_(noise(mlp[2].weight, (4.0 if name == "mlp_color" else 0.6) * float(mlp[2].weight.std())))
    return m.requires_grad_(True)


def _fit_setup():
    from gaustudio_b200 import renderers
    from gaustudio_b200.camera import orbit_cameras
    r = renderers.make("scaffold_renderer")
    fov = math.radians(50.0)
    cams = [c.to("cuda") for c in orbit_cameras(8, 3.0, 20.0, 96, 72, 2 * math.atan(math.tan(fov / 2) * 96 / 72), fov)]
    target = SS.model(1500, 10, F=16, seed=31, outliers=False, device="cuda")
    with torch.no_grad():
        targets = [r.render(c, target)["render"] for c in cams]
    return r, cams, target, targets


def test_training_the_anchors_lowers_the_loss():
    """200 Adam steps of the MLPs, features, offsets and scales fit perturbed parameters (noise from another seed) to
    a target rendered from the true ones: the L1 loss drops at least 4x (5.4-6.3x over two noise seeds on an H100)."""
    r, cams, target, targets = _fit_setup()
    first, last = _fit(r, cams, targets, _perturbed(target, 32), (0.01, 0.002, 0.005, 0.004))
    print(f"\nscaffold fit: L1 {first:.4g} -> {last:.4g} ({first / last:.1f}x)")
    assert last < first / 4, (first, last)


def test_extract_mesh_with_the_scaffold_renderer():
    from gaustudio_b200 import mesh, renderers
    from gaustudio_b200.camera import orbit_cameras
    r = renderers.make("scaffold_renderer")
    m = SS.model(8000, 10, F=16, seed=41, radius=0.5, shell=True, outliers=False, device="cuda")
    with torch.no_grad():
        m._offset.mul_(0.3)
    fov = math.radians(50.0)
    fx = 2 * math.atan(math.tan(fov / 2) * 128 / 96)
    cams = orbit_cameras(16, 2.0, 20.0, 128, 96, fx, fov) + orbit_cameras(8, 2.0, -40.0, 128, 96, fx, fov)
    vs = 0.02
    with torch.no_grad():
        V, F = mesh.extract_mesh(r, m, cams, voxel_size=vs, sdf_trunc=3 * vs, min_weight=1)
    assert F.shape[0] > 1000, F.shape
    rad = V.norm(dim=1)
    assert float((rad - 0.5).abs().median()) < 1.5 * vs, float((rad - 0.5).abs().median())
