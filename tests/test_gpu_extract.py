"""-m gpu: the extraction post-pass kernels (gsr_masked_bilateral / gsr_extract_normals / gsr_normal_fusion_*)
against the reference's own outputs (tests/golden/extract_golden.npz) and the numpy oracle."""
import os
import types

import numpy as np
import pytest
import torch

import extract_ref64 as R
from oracle import extract_oracle as eo

pytestmark = pytest.mark.gpu
G = np.load(os.path.join(os.path.dirname(__file__), "golden", "extract_golden.npz"))
DEV = "cuda"


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


@pytest.mark.parametrize("case", ["a", "b", "c", "s"])
def test_bilateral_matches_reference(case):
    from gaustudio_b200.extract import masked_bilateral_filter
    kw = {}
    if case == "s":
        kw = dict(sigma_color=float(G["bil_s_sigma"][0]), sigma_space=float(G["bil_s_sigma"][1]))
    f, m = masked_bilateral_filter(cu(G[f"bil_{case}_depth"]), cu(G[f"bil_{case}_mask"]), d=int(G[f"bil_{case}_d"]), **kw)
    assert m.dtype == torch.bool and torch.equal(m.cpu(), torch.from_numpy(G[f"bil_{case}_newmask"].astype(bool)))
    # tolerance: OpenCV's 4096-bin range-kernel table vs direct expf, on a ~2 unit depth range
    np.testing.assert_allclose(f.cpu().numpy(), G[f"bil_{case}_filtered"], rtol=0, atol=5e-6)
    ref = R.bilateral64(G[f"bil_{case}_depth"], G[f"bil_{case}_mask"], int(G[f"bil_{case}_d"]), **kw)
    R.check_bilateral(f.cpu().numpy(), m.cpu().numpy(), ref, G[f"bil_{case}_depth"])


def test_bilateral_full_size_and_edges():
    from gaustudio_b200.extract import masked_bilateral_filter
    g = torch.Generator().manual_seed(5)
    H, W = 1080, 1920
    depth = (2 + torch.rand(H, W, generator=g) * 3).float()
    opacity = torch.rand(H, W, generator=g)
    mask = opacity > 0.1
    f, m = masked_bilateral_filter(depth.to(DEV), mask.to(DEV))
    ref = R.bilateral64(depth.numpy(), mask.numpy())
    R.check_bilateral(f.cpu().numpy(), m.cpu().numpy(), ref, depth.numpy())
    assert torch.equal(f.cpu()[~m.cpu()], depth[~m.cpu()])  # masked-out pixels keep their depth bit for bit
    # nothing valid -> pass-through; d = 1 -> identity up to the normalisation round trip
    f0, m0 = masked_bilateral_filter(depth.to(DEV), torch.zeros(H, W, dtype=torch.bool, device=DEV))
    assert torch.equal(f0.cpu(), depth) and not m0.any()
    f1, m1 = masked_bilateral_filter(depth.to(DEV), torch.ones(H, W, dtype=torch.bool, device=DEV), d=1)
    assert m1.all() and (f1.cpu() - depth).abs().max() < 1e-6
    with pytest.raises(RuntimeError):
        masked_bilateral_filter(depth.to(DEV), mask.to(DEV), d=4)
    with pytest.raises(RuntimeError):
        masked_bilateral_filter(depth, mask)  # no CPU path


def _scene(W=160, H=120, P=20000, K=6):
    from gaustudio_b200 import renderers
    from gaustudio_b200.synthetic import build_config
    model, cams, c = build_config("cfg1", P=P, W=W, H=H, K=K)
    model.to(torch.device(DEV))
    return model, cams, renderers.make({"name": "vanilla_renderer"})


def test_extract_view_matches_oracle():
    from gaustudio_b200 import extract
    model, cams, r = _scene()
    radius = extract.getNerfppNorm(cams)["radius"]
    cam = cams[1].to(torch.device(DEV))
    with torch.no_grad():
        pkg = r.render(cam, model)
    v = extract.extract_view(cam, pkg, radius)
    op = pkg["rendered_final_opacity"][0].cpu().numpy(); dp = pkg["rendered_depth"][0].cpu().numpy()
    md = pkg["rendered_median_depth"][0].cpu().numpy(); mi = pkg["rendered_median_id"][0].cpu().numpy()
    K = cam.intrinsics
    E = cam.extrinsics.cpu().numpy()
    ref = R.bilateral64(dp, op > np.float32(0.1))
    mo = ref["new_mask"]
    R.check_bilateral(v["filtered_depth"].cpu().numpy(), v["fg_mask"].cpu().numpy(), ref, dp)
    assert 0.05 < mo.mean() < 1.0
    # normals stage on the SAME filtered depth (the device one), so thresholds see identical inputs
    filt = v["filtered_depth"].cpu().numpy()
    o = eo.view_normals(filt, mo, op, md, mi, float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), E, radius)
    rot = np.linalg.inv(extract._extrinsics_host(cam)[:3, :3]).T.astype(np.float32)   # what extract_view uploads
    r64 = R.view_normals64(filt, mo, op, md, float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), rot,
                           np.float32(radius * 0.8))
    R.close("extract_normals: camera", v["cam_normals"].cpu().numpy(), r64["cam"], r64["A_cam"])
    valid = v["valid"].cpu().numpy()
    R.exact("extract_normals: valid", valid, r64["valid"])
    assert valid.sum() > 100
    edge = np.abs(o["world_sum"] + 3) < 1e-4  # the oracle's float32 sum(world) > -3 may round the other way on the fill
    assert np.array_equal(valid[~edge], o["valid"][~edge])
    R.close("extract_normals: world", v["normals"].cpu().numpy(), r64["neg_world"][valid], r64["A_world"][valid])
    assert np.array_equal(np.sort(v["ids"].cpu().numpy()), np.sort(mi[valid].astype(np.int64)))
    assert torch.equal(v["confidences"].cpu(), torch.from_numpy(op)[v["valid"].cpu()])


def _fusion_inputs():
    V = int(G["fus_V"])
    cams = [types.SimpleNamespace(extrinsics=torch.from_numpy(G[f"fus_E{v}"])) for v in range(V)]
    return (types.SimpleNamespace(_xyz=cu(G["fus_xyz"])), [cu(G[f"fus_ids{v}"]) for v in range(V)],
            [cu(G[f"fus_n{v}"]) for v in range(V)], [cu(G[f"fus_c{v}"]) for v in range(V)], cams)


def test_normal_fusion_matches_reference():
    from gaustudio_b200.extract import normal_fusion
    uid, sm = normal_fusion(*_fusion_inputs())
    assert np.array_equal(uid.cpu().numpy(), G["fus_unique_ids"])
    ref, got = G["fus_smoothed"], sm.cpu().numpy()
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    np.testing.assert_allclose(np.nan_to_num(got), np.nan_to_num(ref), rtol=0, atol=1e-5)


def test_normal_fusion_passes_match_oracle():
    from gaustudio_b200.extract import normal_fusion
    pcd, ids, nrm, conf, cams = _fusion_inputs()
    uid, mean = normal_fusion(pcd, ids, nrm, conf, cams, smooth=False)
    V = int(G["fus_V"])
    ouid, omean = eo.normal_fusion(G["fus_xyz"], [G[f"fus_ids{v}"] for v in range(V)], [G[f"fus_n{v}"] for v in range(V)],
                                   [G[f"fus_c{v}"] for v in range(V)], [G[f"fus_E{v}"][:3, 3] for v in range(V)],
                                   smooth=False)
    assert np.array_equal(uid.cpu().numpy(), ouid)
    ref = R.fusion64(G["fus_xyz"], [G[f"fus_ids{v}"] for v in range(V)], [G[f"fus_n{v}"] for v in range(V)],
                     [G[f"fus_c{v}"] for v in range(V)], [G[f"fus_E{v}"][:3, 3] for v in range(V)])
    assert np.array_equal(ref["uid"], ouid) and ref["p2"]["n_flagged"] == 0
    R.check_mean("fusion: mean", mean.cpu().numpy(), ref["mean2"][ouid], ref["A2"][ouid])


def test_extract_pcd_end_to_end():
    """Render -> filter -> normals -> fusion over an orbit; fused normals of a ball of splats point outwards."""
    from gaustudio_b200 import extract
    model, cams, r = _scene(P=30000, K=8)
    cams = [c.to(torch.device(DEV)) for c in cams]
    xyz, rgb, normals, views = extract.extract_pcd(r, model, cams)
    assert xyz.shape == normals.shape == rgb.shape and xyz.shape[0] > 500
    assert rgb.min() >= 0 and rgb.max() <= 1
    ok = ~torch.isnan(normals).any(1)
    assert ok.float().mean() > 0.5
    assert torch.allclose(normals[ok].norm(dim=1), torch.ones(int(ok.sum()), device=DEV), atol=1e-4)
    # per-view lists agree with the oracle's count for one view (same kernels as test_extract_view_matches_oracle)
    # (the loop runs sync-free: dense per-pixel lists, -1 where the pixel is not a valid observation)
    assert all(int((v["ids"] >= 0).sum()) == int(v["valid"].sum()) and v["ids"].numel() == v["valid"].numel() for v in views)


def test_dense_views_fuse_like_compact_views_and_negative_ids_are_skipped():
    """`extract_view(compact=False)` (no boolean-mask gather, no per-view synchronisation) must fuse to the same
    result as the reference-shaped compact lists; an id of -1 anywhere is "no observation"."""
    from gaustudio_b200 import extract
    model, cams, r = _scene(P=20000, K=5)
    cams = [c.to(torch.device(DEV)) for c in cams]
    radius = extract.getNerfppNorm(cams)["radius"]
    lists = {True: ([], [], []), False: ([], [], [])}
    for cam in cams:
        with torch.no_grad():
            pkg = r.render(cam, model)
        for compact in (True, False):
            v = extract.extract_view(cam, pkg, radius, compact=compact)
            for dst, k in zip(lists[compact], ("ids", "normals", "confidences")):
                dst.append(v[k])
    ua, na = extract.normal_fusion(model, *lists[True], cams, smooth=False)
    ub, nb = extract.normal_fusion(model, *lists[False], cams, smooth=False)
    assert torch.equal(ua, ub) and ua.numel() > 100
    assert torch.equal(torch.isnan(na), torch.isnan(nb))
    assert torch.allclose(torch.nan_to_num(na), torch.nan_to_num(nb), atol=1e-5)
    # a stray -1 in a compact list changes nothing
    ids0 = torch.cat([lists[True][0][0], torch.tensor([-1], device=DEV)])
    n0 = torch.cat([lists[True][1][0], torch.ones(1, 3, device=DEV)])
    c0 = torch.cat([lists[True][2][0], torch.ones(1, device=DEV)])
    uc, nc = extract.normal_fusion(model, [ids0] + lists[True][0][1:], [n0] + lists[True][1][1:], [c0] + lists[True][2][1:],
                                   cams, smooth=False)
    assert torch.equal(ua, uc) and torch.allclose(torch.nan_to_num(na), torch.nan_to_num(nc), atol=1e-6)


@pytest.mark.parametrize("n,shape", [(5000, "ball"), (40000, "shell"), (300, "line")])
def test_device_knn_matches_ckdtree(n, shape):
    """The neighbour search of the fusion's smoothing (extract_pcd.py:170-171, scipy cKDTree there) on the device."""
    from gaustudio_b200.extract import knn
    g = torch.Generator().manual_seed(n)
    p = torch.randn(n, 3, generator=g)
    if shape == "shell":      # a surface: what the extraction produces
        p = p / p.norm(dim=1, keepdim=True) * (1 + 0.01 * torch.randn(n, 1, generator=g))
    elif shape == "line":     # degenerate extents: one cell row
        p = torch.stack([torch.linspace(0, 1, n), torch.zeros(n), torch.zeros(n)], 1) + 1e-4 * p
    p = p.float()
    dist, idx = knn(p.to(DEV), k=10)
    assert torch.equal(idx[:, 0].cpu(), torch.arange(n)) and float(dist[:, 0].abs().max()) == 0.0
    # every neighbour against exact float64 distances (cKDTree on float64 above 6000 points): unique, each distance
    # within rounding, ascending, none missed
    R.check_knn(p.numpy(), dist.cpu().numpy(), idx.cpu().numpy(), 10)
    # unusual k / tiny inputs take the exact all-pairs path
    d3, i3 = knn(p[:7].to(DEV), k=10)
    assert d3.shape == (7, 7) and torch.equal(i3[:, 0].cpu(), torch.arange(7))
