"""Scaffold-GS without a GPU: the float64 restatement of the reference's decoding against a per-anchor, per-offset loop,
the feature-bank mixing, the model's construction checks, the checkpoint round trip, the renderer's refusals and the
argument checks of the new C entry points."""
import os

import pytest
import torch
from torch import nn

import scaffold_ref64 as SR
import scaffold_scenes as SS
from test_abi import _call
from gaustudio_b200 import _lib


def _loop(vis, anchor, offset, scaling, opacity, color, cov):
    """The decoding written per anchor and per offset, from the reference's definition."""
    k = offset.shape[1]
    rows = []
    for i, v in enumerate(vis.tolist()):
        S = scaling[v]
        for j in range(k):
            o = float(opacity[i, j])
            if not o > 0.0:
                continue
            xyz = anchor[v] + offset[v, j] * S[:3]
            rgb = color[i, 3 * j:3 * j + 3]
            s = cov[i, 7 * j:7 * j + 7]
            sc = S[3:] * torch.sigmoid(s[:3])
            q = s[3:7]
            rot = q / max(float(q.norm()), 1e-12)
            rows.append((v, j, xyz, rgb, o, sc, rot))
    return rows


@pytest.mark.parametrize("k", [1, 10, 32])
def test_restatement_matches_a_per_offset_loop(k):
    c = {n: (t.double() if t.is_floating_point() else t) for n, t in SS.decode_case(300, k, 10 + k).items()}
    xyz, rgb, op, sc, rot, mask = SR.decode(**c)
    rows = _loop(**c)
    assert len(rows) == xyz.shape[0] == int(mask.sum())
    assert 0 < len(rows) < c["opacity"].numel()
    # the rows are anchor-major, offset-minor: the mask order
    order = [(int(c["vis"][i]), j) for i, j in zip(*torch.nonzero(mask.view(-1, k), as_tuple=True))]
    assert order == [(v, j) for v, j, *_ in rows]
    ref = [torch.stack([r[n] if torch.is_tensor(r[n]) else torch.tensor([r[n]], dtype=torch.float64) for r in rows])
           for n in (2, 3, 4, 5, 6)]
    for a, b in zip((xyz, rgb, op, sc, rot), ref):
        assert torch.allclose(a, b.reshape(a.shape), rtol=0, atol=1e-12)
    # anchors with all, none and some offsets kept, and exact zeros dropped
    kept = mask.view(-1, k)
    assert bool(kept[0].all()) and not bool(kept[1].any())
    if k > 1:
        assert not bool(kept[2, ::2].any())


def test_feature_bank_mixing_tiles_rather_than_interleaves():
    from gaustudio_b200.scaffold import mix_feature_bank
    g = torch.Generator().manual_seed(3)
    F = 16
    feat = torch.randn(7, F, generator=g, dtype=torch.float64)
    w = torch.softmax(torch.randn(7, 3, generator=g, dtype=torch.float64), 1)
    ref = SR.mix_feature_bank(feat, w)
    ours = mix_feature_bank(feat, w)
    assert torch.allclose(ours, ref, rtol=0, atol=1e-12)
    j = torch.arange(F)
    formula = feat[:, 4 * (j % (F // 4))] * w[:, :1] + feat[:, 2 * (j % (F // 2))] * w[:, 1:2] + feat * w[:, 2:]
    assert torch.allclose(ref, formula, rtol=0, atol=1e-12)
    interleaved = feat[:, ::4].repeat_interleave(4, 1) * w[:, :1] + feat[:, ::2].repeat_interleave(2, 1) * w[:, 1:2] + \
        feat * w[:, 2:]
    assert float((interleaved - ref).abs().max()) > 1e-3


def test_mlp_outputs_use_the_reference_inputs():
    """mlp_outputs builds [feat (bank-mixed), view, dist] as the reference does, and slices off dist for F+3 MLPs."""
    from gaustudio_b200 import scaffold
    for bank, use_dist in ((True, True), (False, False), (True, False)):
        m = SS.model(64, 4, F=8, seed=5, use_feat_bank=bank, use_dist=use_dist)
        cam = SS.camera()
        vis = torch.arange(10, 40)
        o, c, s = scaffold.mlp_outputs(m, vis, cam.camera_center)
        a, f = m._anchor[vis], m._anchor_feat[vis]
        view = a - cam.camera_center
        dist = view.norm(dim=1, keepdim=True)
        view = view / dist
        if bank:
            f = SR.mix_feature_bank(f, m.mlp_feature_bank(torch.cat([view, dist], 1) if use_dist else view))
        inp = torch.cat([f, view, dist], 1) if use_dist else torch.cat([f, view], 1)
        assert torch.equal(o, m.mlp_opacity(inp)) and torch.equal(c, m.mlp_color(inp)) and torch.equal(s, m.mlp_cov(inp))
        assert o.shape == (30, 4) and c.shape == (30, 12) and s.shape == (30, 28)


def _parts(N=5, k=3, F=8, bank=False, dist=True):
    from gaustudio_b200.scaffold import make_mlps
    return [torch.zeros(N, 3), torch.zeros(N, k, 3), torch.zeros(N, F), torch.zeros(N, 1), torch.zeros(N, 6),
            torch.zeros(N, 4)], make_mlps(F, k, bank, dist)


def test_model_refuses_malformed_configurations():
    from gaustudio_b200.scaffold import ScaffoldPointCloud, make_mlps
    t, mlps = _parts()
    ScaffoldPointCloud(*t, **mlps)  # well-formed
    t2, m2 = _parts(bank=True, dist=False)
    ScaffoldPointCloud(*t2, **m2)
    for k in (0, 33):
        tk, mk = _parts(k=max(k, 1))
        tk[1] = torch.zeros(5, k, 3)
        with pytest.raises(ValueError, match="n_offsets"):
            ScaffoldPointCloud(*tk, **make_mlps(8, max(k, 1)))
    tb, mb = _parts(F=6, bank=True)
    with pytest.raises(ValueError, match="multiple of 4"):
        ScaffoldPointCloud(*tb, **mb)
    # an MLP whose widths do not fit F and k, or an appearance embedding's extra inputs
    t, mlps = _parts()
    bad = dict(mlps, mlp_color=nn.Sequential(nn.Linear(8 + 4 + 16, 8), nn.ReLU(), nn.Linear(8, 9), nn.Sigmoid()))
    with pytest.raises(ValueError, match="mlp_color takes 28 inputs"):
        ScaffoldPointCloud(*t, **bad)
    bad = dict(mlps, mlp_cov=nn.Sequential(nn.Linear(12, 8), nn.ReLU(), nn.Linear(8, 20)))
    with pytest.raises(ValueError, match="mlp_cov has 20 outputs"):
        ScaffoldPointCloud(*t, **bad)
    bad = dict(mlps, mlp_opacity=nn.Sequential(nn.Linear(12, 8), nn.ReLU(), nn.Linear(8, 4), nn.Tanh()))
    with pytest.raises(ValueError, match="mlp_opacity has 4 outputs"):
        ScaffoldPointCloud(*t, **bad)
    bad = dict(mlps, mlp_feature_bank=nn.Sequential(nn.Linear(5, 8), nn.ReLU(), nn.Linear(8, 3), nn.Softmax(dim=1)))
    with pytest.raises(ValueError, match="mlp_feature_bank takes 5 inputs"):
        ScaffoldPointCloud(*t, **bad)
    bad = dict(mlps, mlp_opacity=nn.Linear(12, 3))
    with pytest.raises(ValueError, match="nn.Sequential"):
        ScaffoldPointCloud(*t, **bad)


def test_get_attribute_activations():
    import torch.nn.functional as F
    m = SS.model(20, 3, F=8, seed=1)
    assert torch.equal(m.get_attribute("scale"), torch.exp(m._scale))
    assert torch.equal(m.get_attribute("opacity"), torch.sigmoid(m._opacity))
    assert torch.equal(m.get_attribute("rot"), F.normalize(m._rot))
    assert m.get_attribute("mlp_cov") is m.mlp_cov
    assert m.get_attribute("offset") is m._offset and m.get_attribute("anchor") is m._anchor
    m.eval()
    assert not m.mlp_color.training
    m.train()
    assert m.mlp_color.training


@pytest.mark.parametrize("bank", [False, True])
def test_checkpoint_round_trip_is_bit_exact(tmp_path, bank):
    from gaustudio_b200 import io
    m = SS.model(50, 5, F=12, seed=7, use_feat_bank=bank)
    path = str(tmp_path / "point_cloud.ply")
    io.export_scaffold(m, path)
    names = sorted(os.listdir(tmp_path))
    assert names == sorted(["point_cloud.ply", "opacity_mlp.pt", "cov_mlp.pt", "color_mlp.pt"] +
                           (["feature_bank_mlp.pt"] if bank else []))
    # offsets are stored channel-major: f_offset_{c*k+j} is channel c of offset j
    v = io.read_ply_vertices(path)
    assert float(v["f_offset_6"][4]) == float(m._offset[4, 1, 1])  # c = 1, j = 1, k = 5
    back = io.load_scaffold(path)
    for a in ("_anchor", "_offset", "_anchor_feat", "_opacity", "_scale", "_rot"):
        assert torch.equal(getattr(back, a), getattr(m, a)), a
    assert back.n_offsets == 5 and back.feat_dim == 12 and back.use_feat_bank == bank
    x = torch.randn(9, 16)
    for name, mlp in m.mlps().items():
        other = back.mlps()[name]
        assert [type(l) for l in other] == [type(l) for l in mlp], name
        for (ka, va), (kb, vb) in zip(mlp.state_dict().items(), other.state_dict().items()):
            assert ka == kb and torch.equal(va, vb), (name, ka)
        xin = x[:, :mlp[0].in_features]
        assert torch.equal(mlp(xin), other(xin)), name
    # the MLP files may live elsewhere
    (tmp_path / "mlps").mkdir()
    for f in os.listdir(tmp_path):
        if f.endswith(".pt"):
            os.replace(tmp_path / f, tmp_path / "mlps" / f)
    again = io.load_scaffold(path, mlp_dir=str(tmp_path / "mlps"))
    assert torch.equal(again._offset, m._offset)
    with pytest.raises(FileNotFoundError):
        io.load_scaffold(path)


def test_renderer_refuses_subpixel_offset_and_bad_kernel_size():
    from gaustudio_b200 import renderers
    r = renderers.make("scaffold_renderer")
    assert r.kernel_size == 0.0 and r.scaling_modifier == 1.0 and not r.white_background
    assert r.bg_color.device.type == "cpu"
    m = SS.model(10, 2, F=8)
    with pytest.raises(NotImplementedError, match="subpixel_offset"):
        r.render(SS.camera(), m, subpixel_offset=torch.zeros(SS.H, SS.W, 2))
    with pytest.raises(ValueError, match="kernel_size"):
        renderers.make({"name": "scaffold_renderer", "kernel_size": -1.0})
    renderers.make({"name": "scaffold_renderer", "convert_SHs_python": True, "compute_cov3D_python": True})


def test_entry_points_refuse_bad_arguments_before_any_work():
    K = "gsr_scaffold_count: Nv >= 0 and 1 <= k <= 32"
    for k in (0, 33, -1):
        assert _call("gsr_scaffold_count", Nv=10, k=k) == -1 and _lib.last_error() == K
    assert _call("gsr_scaffold_count", Nv=-1, k=4) == -1 and _lib.last_error() == K
    assert _call("gsr_scaffold_count", Nv=1 << 27, k=32) == -1 and "int32" in _lib.last_error()
    assert _call("gsr_scaffold_count", Nv=10, k=4, opacity=None) == -1 and "null" in _lib.last_error()
    for k in (0, 33):
        assert _call("gsr_scaffold_decode", Nv=10, k=k) == -1
        assert _lib.last_error() == "gsr_scaffold_decode: Nv >= 0 and 1 <= k <= 32"
        assert _call("gsr_scaffold_decode_backward", N=20, Nv=10, k=k) == -1
    assert _call("gsr_scaffold_decode_backward", N=5, Nv=10, k=4) == -1
    assert _lib.last_error() == "gsr_scaffold_decode_backward: 0 <= Nv <= N and 1 <= k <= 32"
    assert _call("gsr_scaffold_decode", Nv=0, k=4) == 0  # nothing to do
    assert _call("gsr_scaffold_decode", Nv=10, k=4, rotations=(1 << 20) + 4) == -1
    assert _lib.last_error() == "gsr_scaffold_decode: rotations must be 16-byte aligned"
    assert _call("gsr_scaffold_visible", N=10, kernel_size=-0.1) == -1
    assert _lib.last_error() == "gsr_scaffold_visible: kernel_size must be finite and >= 0"
    assert _call("gsr_scaffold_visible", N=10, kernel_size=float("inf")) == -1
    assert _call("gsr_scaffold_visible", N=10, width=0) == -1
    assert _call("gsr_scaffold_visible", N=10, cov3D_precomp=None, scales=None) == -1
    assert _call("gsr_scaffold_visible", N=10, cov3D_precomp=None, rotations=(1 << 20) + 8) == -1
    assert _lib.last_error() == "gsr_scaffold_visible: rotations must be 16-byte aligned"
    assert _call("gsr_scaffold_visible", N=0) == 0
