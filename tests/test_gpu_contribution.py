"""-m gpu: the contribution statistics (gsr_contribution, gaustudio_b200.prune) against float64 and against the forward.

1. Per Gaussian against tests/contrib_ref64.py, built from the forward's exported state: count exact and weight /
   max_weight within the derived bound for every Gaussian no ambiguous pixel could reach; scenes A-D, a dense and a
   sparse scene, an image wider than one tile-scan round; the un-fused, fused and Mip (k = 0.1, 0.3) paths.
2. Invariants: per view the weights sum to the opacity image within a derived bound; V views accumulated equal the
   float64 sum of V one-view passes exactly.
3. Prune invariance: removing every Gaussian with count == 0 over a set of views leaves those views' colour, depth,
   opacity, median depth and weight bit-identical, the median ids equal through the kept-index map and the kept radii
   identical, on all three paths.  Any blend or termination decision of the pass that differed from the forward's
   would break this.
4. Determinism: same bits across repeated passes, speculation on and off, every tile order, pipelined mode, and after
   another scene used the buffers.
5. prune with FusedAdam state, filter_3D and the densification statistics; the PLY round trip; a cfg 1 model pruned at
   ratio 0.5.
6. Refusals."""

import numpy as np
import pytest
import torch

import comp_ref64 as R
import contrib_ref64 as CR
import scenes
from test_gpu_compositing_f64 import view_scene

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
U = 2.0 ** -24


def raw_forward(s):
    """_C.rasterize_gaussians on a scenes.scene-format dict -> its 9-tuple."""
    from gaustudio_b200 import _C
    e = torch.Tensor([])
    d = lambda k: torch.as_tensor(s[k]).to(DEV).contiguous() if s.get(k) is not None else e
    cam = [torch.as_tensor(np.asarray(s[k], np.float32)).to(DEV) for k in ("viewmatrix", "projmatrix", "campos")]
    return _C.rasterize_gaussians(torch.as_tensor(s["bg"]).to(DEV), d("means3D"), d("colors_precomp"), d("opacities"),
                                  d("scales"), d("rotations"), s["scale_modifier"], d("cov3D_precomp"), cam[0], cam[1],
                                  s["tanfovx"], s["tanfovy"], s["H"], s["W"], d("shs"), s["D"], cam[2], False, False)


def accumulators(P):
    return (torch.zeros(P, dtype=torch.float64, device=DEV), torch.zeros(P, dtype=torch.int64, device=DEV),
            torch.zeros(P, dtype=torch.float32, device=DEV))


def run_pass(out, P, H, W, acc=None):
    from gaustudio_b200 import _C
    acc = accumulators(P) if acc is None else acc
    _C.contribution(P, H, W, out[6], out[0], out[7], out[8], *acc)
    return acc


def reference(out, P, H, W):
    from gaustudio_b200 import _C
    ex = _C.debug_export(P, W, H, out[0], out[6], out[7], out[8])
    ex = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in ex.items()}
    comp = R.Compositing(ex["means2D"], ex["conic_opacity"], ex["rgb"], ex["depths"], out[5].cpu(), W, H, np.zeros(3))
    return comp, ex


def compare(acc, st, what):
    weight, count, maxw = (t.cpu() for t in acc)
    ok = ~st.tainted
    reached = st.count > 0
    assert int((ok & reached).sum()) >= 0.5 * int(reached.sum()), f"{what}: too few unambiguous Gaussians"
    bad = ok & (count != st.count)
    assert not bad.any(), f"{what}: count differs for {int(bad.sum())} Gaussians"
    ew = (weight - st.weight).abs()
    bad = ok & (ew > st.weight_bound())
    assert not bad.any(), f"{what}: weight beyond bound for {int(bad.sum())}, worst {float(ew[ok].max()):.3e}"
    em = (maxw.double() - st.max).abs()
    bad = ok & (em > st.max_bound)
    assert not bad.any(), f"{what}: max_weight beyond bound for {int(bad.sum())}, worst {float(em[ok].max()):.3e}"
    assert (count[~reached & ok] == 0).all() and (weight[count == 0] == 0).all() and (maxw[count == 0] == 0).all()


SCENES = {"A": lambda: scenes.scene("A"), "B": lambda: scenes.scene("B"), "C": lambda: scenes.scene("C"),
          "D": lambda: scenes.scene("D"), "dense": lambda: view_scene("saturating", 64, 48, 2),
          "sparse": lambda: view_scene("partial", 250, 170, 4), "wide2561x1441": lambda: view_scene("wide", 2561, 1441, 8)}


@pytest.mark.parametrize("key", list(SCENES))
def test_statistics_against_f64_unfused(key):
    s = SCENES[key]()
    out = raw_forward(s)
    P, H, W = out[5].numel(), s["H"], s["W"]
    acc = run_pass(out, P, H, W)
    comp, _ = reference(out, P, H, W)
    compare(acc, CR.Statistics(P).add(comp), key)


def cfg1(P=4000, K=6, W=128, H=96):
    from gaustudio_b200.synthetic import build_config
    model, cams, _ = build_config("cfg1", P=P, K=K, W=W, H=H)
    model.active_sh_degree = 3
    return model.to(DEV), [c.to(DEV) for c in cams]


def path_setup(path):
    """(model, cameras, renderer) for 'vanilla', 'fused', 'mip0.1' or 'mip0.3'."""
    from gaustudio_b200 import renderers
    from gaustudio_b200.mip import MipPointCloud
    model, cams = cfg1()
    if path == "vanilla":
        return model, cams, renderers.make("vanilla_renderer")
    if path == "fused":
        r = renderers.make({"name": "vanilla_renderer", "fused_activations": True})
        assert r._can_fuse(model)
        return model, cams, r
    m = MipPointCloud.from_model(model)
    m.compute_3D_filter(cams)
    return m, cams, renderers.make({"name": "mip_renderer", "kernel_size": float(path[3:])})


@pytest.mark.parametrize("path", ["vanilla", "fused", "mip0.1", "mip0.3"])
def test_statistics_against_f64_on_every_path(path):
    from gaustudio_b200 import prune as PR
    model, cams, r = path_setup(path)
    P = model._xyz.shape[0]
    st = CR.Statistics(P)
    acc = accumulators(P)
    with torch.no_grad():
        for cam in cams[:3]:
            out, H, W = PR._forward(r, cam, model)
            run_pass(out, P, H, W, acc)
            st.add(reference(out, P, H, W)[0])
    compare(acc, st, path)
    # prune.contribution makes the same forwards and passes
    c = PR.contribution(model, cams[:3], r)
    assert c["views"] == 3
    for got, want in zip((c["weight"], c["count"], c["max_weight"]), acc):
        assert torch.equal(got, want)


def test_invariants():
    s = view_scene("saturating", 64, 48, 2)
    out = raw_forward(s)
    P, H, W = out[5].numel(), s["H"], s["W"]
    weight, count, _ = run_pass(out, P, H, W)
    from gaustudio_b200 import _C
    nc = _C.debug_export(P, W, H, out[0], out[6], out[7], out[8])["n_contrib"].double().sum()
    opac = out[4].double().sum()
    bound = 2.1 * U * float(nc) + U * H * W
    assert abs(float(weight.sum()) - float(opac)) <= bound
    # V views: one accumulation equals the float64 sum, in view order, of V one-view passes
    model, cams, r = path_setup("vanilla")
    from gaustudio_b200 import prune as PR
    whole = PR.contribution(model, cams, r)
    total = torch.zeros_like(whole["weight"])
    cnt = torch.zeros_like(whole["count"])
    mx = torch.zeros_like(whole["max_weight"])
    for cam in cams:
        one = PR.contribution(model, [cam], r)
        total = total + one["weight"]
        cnt += one["count"]
        mx = torch.maximum(mx, one["max_weight"])
    assert torch.equal(whole["weight"], total) and torch.equal(whole["count"], cnt)
    assert torch.equal(whole["max_weight"], mx)


@pytest.mark.parametrize("path", ["vanilla", "fused", "mip0.3"])
def test_pruning_what_no_view_reached_changes_no_bit(path):
    from gaustudio_b200 import prune as PR
    model, cams, r = path_setup(path)
    P = model._xyz.shape[0]
    c = PR.contribution(model, cams, r)
    keep = c["count"] > 0
    n_keep = int(keep.sum())
    assert 0 < n_keep < P, f"{path}: nothing to prune ({n_keep} of {P} kept)"
    with torch.no_grad():
        before = [r.render(cam, model) for cam in cams]
    PR.prune(model, keep)
    assert model._xyz.shape[0] == n_keep
    new_index = torch.cumsum(keep.long(), 0) - 1
    with torch.no_grad():
        after = [r.render(cam, model) for cam in cams]
    for v, (b, a) in enumerate(zip(before, after)):
        for k in ("render", "rendered_depth", "rendered_final_opacity", "rendered_median_depth",
                  "rendered_median_weight"):
            assert torch.equal(b[k], a[k]), f"{path} view {v}: {k} changed"
        has = b["rendered_median_weight"] > 0
        bid, aid = b["rendered_median_id"], a["rendered_median_id"]
        assert torch.equal(aid[~has], bid[~has])
        assert torch.equal(aid[has], new_index[bid[has].long()].int()), f"{path} view {v}: median ids"
        assert keep[bid[has].long()].all()
        assert torch.equal(b["radii"][keep], a["radii"]), f"{path} view {v}: radii"


def test_determinism():
    from gaustudio_b200 import _C
    from gaustudio_b200 import prune as PR
    model, cams, r = path_setup("vanilla")
    first = PR.contribution(model, cams, r)
    same = lambda c: all(torch.equal(c[k], first[k]) for k in ("weight", "count", "max_weight"))
    assert same(PR.contribution(model, cams, r))
    order_prev = _C.set_tile_order(1)
    spec_prev = _C.set_speculation(None)
    try:
        for order in (0, 1, 2):
            _C.set_tile_order(order)
            for spec in (True, False):
                _C.set_speculation(spec)
                assert same(PR.contribution(model, cams, r)), (order, spec)
    finally:
        _C.set_tile_order(order_prev)
        _C.set_speculation(spec_prev)
    state = _C.pipeline_state()
    try:
        _C.set_pipelined(True)
        got = PR.contribution(model, cams + cams, r)  # the second round runs pipelined
        _C.check_pipeline(wait=True)
    finally:
        _C.restore_pipeline(state)
    assert torch.equal(got["count"], 2 * first["count"])
    assert torch.equal(got["max_weight"], first["max_weight"])
    # another scene fills the caching allocator's blocks with its own state first
    other, ocams = cfg1(P=6000, K=2)
    PR.contribution(other, ocams, r)
    assert same(PR.contribution(model, cams, r))


def test_prune_with_optimizer_state_and_ply_round_trip(tmp_path):
    from gaustudio_b200 import io, optimizers, renderers
    from gaustudio_b200 import prune as PR
    m, cams, r = path_setup("mip0.3")
    for a in PR.ATTRS:
        setattr(m, a, torch.nn.Parameter(getattr(m, a).detach().clone()))
    opt = optimizers.FusedAdam(m.parameters_list(), lr=1e-3, eps=1e-15, weight_decay=0.0)
    g = torch.Generator(device=DEV).manual_seed(5)
    for p in m.parameters_list():
        p.grad = torch.randn(p.shape, generator=g, device=DEV)
    opt.step()
    n = m._xyz.shape[0]
    m.xyz_gradient_accum = torch.rand(n, 1, generator=g, device=DEV)
    m.denom = torch.rand(n, 1, generator=g, device=DEV)
    m.max_radii2D = torch.rand(n, generator=g, device=DEV)
    P = m._xyz.shape[0]
    old = {a: getattr(m, a).detach().clone() for a in PR.ATTRS}
    old_st = {a: {k: v.clone() for k, v in opt.state[getattr(m, a)].items() if torch.is_tensor(v)} for a in PR.ATTRS}
    steps = {a: opt.state[getattr(m, a)]["step"] for a in PR.ATTRS}
    old_stats = [t.clone() for t in (m.xyz_gradient_accum, m.denom, m.max_radii2D, m.filter_3D)]
    keep = torch.rand(P, generator=torch.Generator().manual_seed(3)).to(DEV) < 0.6
    idx = keep.nonzero().squeeze(1)
    PR.prune(m, keep, opt)
    for a in PR.ATTRS:
        p = getattr(m, a)
        assert torch.equal(p.detach(), old[a][idx])
        st = opt.state[p]
        assert st["step"] == steps[a]
        for k, v in old_st[a].items():
            assert torch.equal(st[k], v[idx]), (a, k)
    for t, o in zip((m.xyz_gradient_accum, m.denom, m.max_radii2D, m.filter_3D), old_stats):
        assert torch.equal(t, o[idx])
    path = str(tmp_path / "pruned.ply")
    io.export_ply(m, path)
    back = io.load_ply(path, sh_degree=3, device=DEV)
    n = m._xyz.shape[0]
    ply_layout = lambda t: t.detach().reshape(n, -1, 3).transpose(1, 2).reshape(n, -1)  # SH stored channel-major
    for a in PR.ATTRS:
        want = ply_layout(getattr(m, a)) if a in ("_f_dc", "_f_rest") else getattr(m, a).detach()
        assert torch.equal(getattr(back, a).reshape(want.shape), want), a
    assert torch.equal(back.filter_3D, m.filter_3D)
    # cfg 1 at ratio 0.5: exactly floor(P / 2) rows go, the rest still renders
    full, fcams = cfg1(P=None, K=4, W=256, H=256)
    Pf = full._xyz.shape[0]
    vr = renderers.make("vanilla_renderer")
    score = PR.significance(full, PR.contribution(full, fcams, vr))
    res = PR.prune(full, PR.select(score, 0.5))
    assert res["P_after"] == Pf - Pf // 2
    with torch.no_grad():
        for cam in fcams:
            o = vr.render(cam, full)
            assert torch.isfinite(o["render"]).all() and torch.isfinite(o["rendered_depth"]).all()


def test_refusals():
    from gaustudio_b200 import _C, _lib, renderers
    from gaustudio_b200 import prune as PR
    model, cams = cfg1(P=500, K=2)
    for name in ("surfel_renderer", "scaffold_renderer"):
        with pytest.raises(NotImplementedError):
            PR.contribution(model, cams, renderers.make(name))
    with pytest.raises(ValueError, match="no cameras"):
        PR.contribution(model, [], renderers.make("vanilla_renderer"))
    r = renderers.make("vanilla_renderer")
    with torch.no_grad():
        out, H, W = PR._forward(r, cams[0], model)
    w, c, m = accumulators(499)
    with pytest.raises(ValueError, match="shape"):
        _C.contribution(500, H, W, out[6], out[0], out[7], out[8], w, c, m)
    with pytest.raises(ValueError, match="rows"):
        PR.significance(model, dict(weight=w))
    w, c, m = accumulators(500)
    L = _lib.lib()
    assert L.gsr_contribution(500, out[0], W, H, out[6].data_ptr(), out[7].data_ptr(), out[8].data_ptr(), None,
                              c.data_ptr(), m.data_ptr(), None) == -1
    assert "weight, count and max_weight" in _lib.last_error()
    assert L.gsr_contribution(500, out[0], 0, H, out[6].data_ptr(), out[7].data_ptr(), out[8].data_ptr(),
                              w.data_ptr(), c.data_ptr(), m.data_ptr(), None) == -1
    torch.cuda.synchronize()
    assert int(c.sum()) == 0
