"""Contribution-based pruning without a GPU: the float64 statistics of tests/contrib_ref64.py against a scalar per-pixel
loop, LightGaussian's significance formula, the tie rule of `select`, and `prune` on CPU tensors with torch.optim.Adam
state, the densification statistics and a Mip model's filter_3D.  The refusals that happen before any device work."""
import math

import numpy as np
import pytest
import torch

import comp_ref64 as R
import contrib_ref64 as CR
from gaustudio_b200 import prune as PR
from gaustudio_b200.mip import MipPointCloud
from gaustudio_b200.synthetic import make_scene


def splats(seed, W, H, P, opaque):
    """Random 2-D splats over (and a little beyond) a W x H image: means2D, conic_opacity, depths, radii (float32)."""
    rng = np.random.RandomState(seed)
    m2 = np.stack([rng.uniform(-6, W + 6, P), rng.uniform(-6, H + 6, P)], 1)
    sd = rng.uniform(1.0, 7.0, (P, 2))
    th = rng.uniform(0, np.pi, P)
    c, s = np.cos(th), np.sin(th)
    rot = np.stack([np.stack([c, -s], 1), np.stack([s, c], 1)], 1)
    cov = rot @ (sd[:, :, None] ** 2 * np.eye(2)) @ rot.transpose(0, 2, 1)
    inv = np.linalg.inv(cov)
    op = rng.uniform(0.6, 1.0, P) if opaque else rng.uniform(0.002, 0.6, P)
    co = np.stack([inv[:, 0, 0], inv[:, 0, 1], inv[:, 1, 1], op], 1).astype(np.float32)
    radii = np.ceil(3 * np.sqrt(np.linalg.eigvalsh(cov).max(1))).astype(np.int32)
    radii[:3] = 0  # culled by the projection: never in a list
    return m2.astype(np.float32), co, rng.uniform(1, 5, P).astype(np.float32), radii


@pytest.mark.parametrize("seed,W,H,P,opaque", [(0, 40, 24, 60, False), (1, 37, 21, 90, True), (2, 16, 16, 40, True),
                                               (3, 50, 9, 120, False)])
def test_statistics_match_a_per_pixel_loop(seed, W, H, P, opaque):
    m2, co, dep, radii = splats(seed, W, H, P, opaque)
    comp = R.Compositing(m2, co, np.zeros((P, 3)), dep, radii, W, H, np.zeros(3))
    st = CR.Statistics(P).add(comp)
    w, cnt, mx = CR.brute_force(m2, co, dep, radii, W, H)
    assert np.array_equal(st.count.numpy(), cnt)
    np.testing.assert_allclose(st.weight.numpy(), w, rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(st.max.numpy(), mx, rtol=1e-12, atol=0)
    assert (st.count[:3] == 0).all() and (st.weight[:3] == 0).all()
    # an ending pair is counted without weight: count exceeds the blended pixels exactly by the pixels that ended
    assert int(st.count.sum()) == int(comp.n_contrib.sum()) + int(comp.ended.sum())
    if opaque:
        assert int(comp.ended.sum()) > 0
    # blend weights telescope: per pixel sum of w = 1 - T_final
    assert abs(float(st.weight.sum()) - float((1 - comp.final_T).sum())) < 1e-9
    # a Gaussian is tainted exactly when a flagged pixel could have reached it; untainted ones exist
    assert not st.tainted.all()


def test_taint_covers_every_gaussian_a_flagged_pixel_reaches():
    """A pixel flagged for alpha near 1/255 taints the Gaussian that sits on the threshold, and its neighbours behind."""
    W, H = 16, 16
    # Gaussian 0 centred on pixel (3, 3) with o = 1/255 exactly at the centre pixel; Gaussian 1 behind it, opaque
    m2 = np.array([[3.0, 3.0], [3.0, 3.0], [12.0, 12.0]], np.float32)
    co = np.array([[0.5, 0.0, 0.5, 1.0 / 255.0], [0.5, 0.0, 0.5, 0.5], [0.5, 0.0, 0.5, 0.5]], np.float32)
    comp = R.Compositing(m2, co, np.zeros((3, 3)), np.array([1, 2, 3], np.float32), np.array([4, 4, 4]), W, H,
                         np.zeros(3))
    assert bool(comp.flag[3 * W + 3])
    st = CR.Statistics(3).add(comp)
    assert st.tainted[0] and st.tainted[1] and not st.tainted[2]


def model_of(P, seed=0):
    return make_scene(P, 1.0, 0.05, seed, sh_degree=1)


def test_significance_is_lightgaussians_volume_weighted_score():
    m = model_of(50)
    g = torch.Generator().manual_seed(1)
    w = torch.rand(50, generator=g, dtype=torch.float64)
    contrib = dict(weight=w, count=torch.ones(50, dtype=torch.int64), max_weight=w.float(), views=1)
    s = torch.exp(m._scale.double())
    V = s[:, 0] * s[:, 1] * s[:, 2]
    v_ref = sorted(V.tolist(), reverse=True)[int(0.9 * 50)]
    want = w * (V / v_ref) ** 0.1
    got = PR.significance(m, contrib)
    assert got.dtype == torch.float64
    torch.testing.assert_close(got, want, rtol=1e-6, atol=0)  # V from float32 activated scales
    torch.testing.assert_close(PR.significance(m, contrib, v_pow=0.5), w * (V / v_ref) ** 0.5, rtol=1e-6, atol=0)
    # the reference volume ranks at floor(0.9 P) in descending order: score == weight there
    i = int(torch.argsort(V, descending=True, stable=True)[45])
    assert abs(float(got[i]) - float(w[i])) <= 1e-6 * float(w[i])
    with pytest.raises(ValueError, match="rows"):
        PR.significance(model_of(49), contrib)


def test_significance_uses_the_filtered_scales_of_a_mip_model():
    base = model_of(40)
    f = torch.full((40, 1), 0.07)
    m = MipPointCloud.from_model(base, filter_3D=f)
    contrib = dict(weight=torch.ones(40, dtype=torch.float64))
    sf = torch.sqrt(torch.exp(base._scale.double()) ** 2 + 0.07 ** 2)
    V = sf.prod(1)
    v_ref = torch.sort(V, descending=True).values[36]
    torch.testing.assert_close(PR.significance(m, contrib), (V / v_ref) ** 0.1, rtol=1e-6, atol=0)


def test_select_keeps_an_exact_count_with_ties_to_the_lower_index():
    score = torch.tensor([3.0, 1.0, 2.0, 2.0, 2.0, 0.0, 5.0, 2.0], dtype=torch.float64)
    keep = PR.select(score, 0.5)  # drop floor(4) = 4: keep 5.0, 3.0 and the first two 2.0s
    assert keep.tolist() == [True, False, True, True, False, False, True, False]
    for r in (0.0, 0.1, 0.33, 0.5, 0.66, 0.999, 1.0):
        assert int(PR.select(score, r).sum()) == 8 - math.floor(r * 8)
    assert PR.select(torch.zeros(7, dtype=torch.float64), 3 / 7).tolist() == [True] * 4 + [False] * 3
    with pytest.raises(ValueError):
        PR.select(score, 1.5)
    with pytest.raises(ValueError):
        PR.select(score, -0.1)


def _adam_model(P):
    m = model_of(P)
    for a in PR.ATTRS:
        setattr(m, a, torch.nn.Parameter(getattr(m, a).clone()))
    opt = torch.optim.Adam(m.parameters_list(), lr=1e-3)
    loss = sum((p * (i + 1)).square().sum() for i, p in enumerate(m.parameters_list()))
    loss.backward()
    opt.step()
    return m, opt


def test_prune_compacts_rows_and_adam_state_in_order():
    P = 30
    m, opt = _adam_model(P)
    m.xyz_gradient_accum = torch.arange(P, dtype=torch.float32)[:, None]
    m.denom = 2 * torch.arange(P, dtype=torch.float32)[:, None]
    m.max_radii2D = 3 * torch.arange(P, dtype=torch.float32)
    old = {a: getattr(m, a).detach().clone() for a in PR.ATTRS}
    old_state = {a: {k: (v.clone() if torch.is_tensor(v) else v) for k, v in opt.state[getattr(m, a)].items()}
                 for a in PR.ATTRS}
    keep = torch.zeros(P, dtype=torch.bool)
    keep[[0, 3, 4, 17, 29]] = True
    idx = keep.nonzero().squeeze(1)
    res = PR.prune(m, keep, opt)
    assert res == dict(P_before=P, P_after=5, pruned=P - 5)
    assert m.num_points == 5
    for a in PR.ATTRS:
        p = getattr(m, a)
        assert isinstance(p, torch.nn.Parameter) and p.requires_grad
        assert torch.equal(p.detach(), old[a][idx])
        assert any(q is p for g in opt.param_groups for q in g["params"])
        st = opt.state[p]
        assert torch.equal(st["exp_avg"], old_state[a]["exp_avg"][idx])
        assert torch.equal(st["exp_avg_sq"], old_state[a]["exp_avg_sq"][idx])
        assert torch.equal(st["step"], old_state[a]["step"])  # the step count is kept
    assert len(opt.state) == len(PR.ATTRS)
    assert torch.equal(m.xyz_gradient_accum[:, 0], idx.float())
    assert torch.equal(m.denom[:, 0], 2 * idx.float())
    assert torch.equal(m.max_radii2D, 3 * idx.float())
    # the optimizer keeps working on the pruned parameters
    sum(p.square().sum() for p in m.parameters_list()).backward()
    opt.step()


def test_prune_a_mip_model_keeps_filter_3D_with_its_rows():
    base = model_of(12)
    m = MipPointCloud.from_model(base, filter_3D=torch.arange(12, dtype=torch.float32))
    keep = torch.tensor([i % 3 != 1 for i in range(12)])
    PR.prune(m, keep)
    assert torch.equal(m.filter_3D[:, 0], torch.tensor([0., 2, 3, 5, 6, 8, 9, 11]))
    assert m._xyz.shape[0] == 8 and m.get_scaling_with_3D_filter.shape == (8, 3)
    PR.prune(m, torch.ones(8, dtype=torch.bool))  # keep everything: unchanged
    assert m._xyz.shape[0] == 8
    PR.prune(m, torch.zeros(8, dtype=torch.bool))
    assert m._xyz.shape[0] == 0 and m.filter_3D.shape == (0, 1)


def test_prune_refusals():
    import scaffold_scenes
    m = model_of(10)
    with pytest.raises(ValueError, match="bool"):
        PR.prune(m, torch.ones(10, dtype=torch.int64))
    with pytest.raises(ValueError, match="shape"):
        PR.prune(m, torch.ones(9, dtype=torch.bool))
    with pytest.raises(NotImplementedError):
        PR.prune(scaffold_scenes.model(8, 4), torch.ones(8, dtype=torch.bool))
    assert m._xyz.shape[0] == 10


def test_contribution_refusals_come_before_any_device_work():
    import scaffold_scenes
    from gaustudio_b200 import renderers
    from gaustudio_b200.camera import orbit_cameras
    m = model_of(10)  # a CPU model: any device work would fail differently
    cams = orbit_cameras(2, 3.0, 30.0, 32, 32, 0.8, 0.8)
    for name in ("surfel_renderer", "scaffold_renderer"):
        with pytest.raises(NotImplementedError):
            PR.contribution(m, cams, renderers.make(name))
    with pytest.raises(NotImplementedError):
        PR.contribution(scaffold_scenes.model(8, 4), cams, renderers.make("scaffold_renderer"))
    with pytest.raises(ValueError, match="no cameras"):
        PR.contribution(m, [], renderers.make("vanilla_renderer"))
    with pytest.raises(ValueError, match="filter_3D"):
        PR.contribution(MipPointCloud.from_model(m), cams, renderers.make("mip_renderer"))
    with pytest.raises(RuntimeError, match="CUDA"):
        PR.contribution(m, cams, renderers.make("vanilla_renderer"))
