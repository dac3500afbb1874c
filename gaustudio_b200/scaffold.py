"""ScaffoldPointCloud: the anchor model of Scaffold-GS (gaustudio's `scaffold_pcd`, `models/scaffold_sg.py`), and the
neural-Gaussian decoding the `scaffold_renderer` runs on every view.

An anchor carries a position `_anchor [N,3]`, k learnable offsets `_offset [N,k,3]`, a feature `_anchor_feat [N,F]`,
six log-scales `_scale [N,6]` (three scale the offsets, three the neural Gaussians) and `_rot [N,4]`.  Three MLPs
(optionally four) turn a visible anchor's feature, viewing direction and distance into the opacities, colours and
covariances of its k neural Gaussians.  The MLPs stay in torch (cuBLAS GEMMs, autograd); what follows them -- the
compaction of the Gaussians with opacity > 0 and their attributes -- is one CUDA decode and one CUDA backward
(include/gsr.h, gsr_scaffold_decode).  Differences from the reference model, which cannot be constructed: the typo in
`use_feat_bank`, the print in `get_attribute` and the device hard-coded in the MLPs are gone.
"""
import torch
import torch.nn.functional as F
from torch import nn

from . import _C

MAX_OFFSETS = 32


def make_mlps(feat_dim, n_offsets, use_feat_bank=False, use_dist=True):
    """The reference's MLPs (scaffold_sg.py:49-76): Linear -> ReLU -> Linear, then Tanh (opacity), nothing (cov),
    Sigmoid (colour), Softmax(dim=1) (feature bank).  use_dist: the inputs end with the anchor's distance to the
    camera (F+4 inputs, the reference's layout) instead of only the viewing direction (F+3)."""
    d = feat_dim + 3 + int(use_dist)
    mlps = dict(
        mlp_opacity=nn.Sequential(nn.Linear(d, feat_dim), nn.ReLU(True), nn.Linear(feat_dim, n_offsets), nn.Tanh()),
        mlp_cov=nn.Sequential(nn.Linear(d, feat_dim), nn.ReLU(True), nn.Linear(feat_dim, 7 * n_offsets)),
        mlp_color=nn.Sequential(nn.Linear(d, feat_dim), nn.ReLU(True), nn.Linear(feat_dim, 3 * n_offsets),
                                nn.Sigmoid()))
    if use_feat_bank:
        mlps["mlp_feature_bank"] = nn.Sequential(nn.Linear(3 + int(use_dist), feat_dim), nn.ReLU(True),
                                                 nn.Linear(feat_dim, 3), nn.Softmax(dim=1))
    return mlps


def _widths(name, mlp):
    if not (isinstance(mlp, nn.Sequential) and len(mlp) >= 3 and isinstance(mlp[0], nn.Linear)
            and isinstance(mlp[2], nn.Linear) and mlp[0].out_features == mlp[2].in_features):
        raise ValueError(f"{name} must be an nn.Sequential of Linear, ReLU, Linear[, activation]")
    return mlp[0].in_features, mlp[2].out_features


class ScaffoldPointCloud(nn.Module):
    activations = {"scale": torch.exp, "opacity": torch.sigmoid, "rot": lambda r: F.normalize(r)}
    _ATTRS = ("_anchor", "_offset", "_anchor_feat", "_opacity", "_scale", "_rot")

    def __init__(self, anchor, offset, anchor_feat, opacity, scale, rot, mlp_opacity, mlp_cov, mlp_color,
                 mlp_feature_bank=None):
        super().__init__()
        N = anchor.shape[0]
        if offset.dim() != 3 or offset.shape[0] != N or offset.shape[2] != 3:
            raise ValueError(f"offset must be [N,k,3], got {tuple(offset.shape)}")
        k, Fd = offset.shape[1], anchor_feat.shape[-1]
        if not 1 <= k <= MAX_OFFSETS:
            raise ValueError(f"n_offsets must be 1..{MAX_OFFSETS}, got {k}")
        if tuple(anchor.shape) != (N, 3) or tuple(anchor_feat.shape) != (N, Fd) or tuple(scale.shape) != (N, 6) or \
                tuple(rot.shape) != (N, 4) or opacity.numel() != N:
            raise ValueError("anchor [N,3], anchor_feat [N,F], opacity [N,1], scale [N,6] and rot [N,4] must agree")
        self.use_feat_bank = mlp_feature_bank is not None
        if self.use_feat_bank and Fd % 4 != 0:
            raise ValueError(f"the feature bank mixes F/4, F/2 and F channels: feat_dim must be a multiple of 4, got {Fd}")
        for name, mlp, out in (("mlp_opacity", mlp_opacity, k), ("mlp_cov", mlp_cov, 7 * k),
                               ("mlp_color", mlp_color, 3 * k), ("mlp_feature_bank", mlp_feature_bank, 3)):
            if mlp is None:
                continue
            din, dout = _widths(name, mlp)
            ok_in = (3, 4) if name == "mlp_feature_bank" else (Fd + 3, Fd + 4)
            if din not in ok_in:
                raise ValueError(f"{name} takes {din} inputs; it must take {ok_in[1]} ([feat, view, dist]) or "
                                 f"{ok_in[0]} (without dist) -- appearance embeddings are not supported")
            if dout != out:
                raise ValueError(f"{name} has {dout} outputs; with {k} offsets it must have {out}")
        self._anchor, self._offset, self._anchor_feat = anchor, offset, anchor_feat
        self._opacity, self._scale, self._rot = opacity.reshape(N, 1), scale, rot
        self.mlp_opacity, self.mlp_cov, self.mlp_color = mlp_opacity, mlp_cov, mlp_color
        self.mlp_feature_bank = mlp_feature_bank
        self.n_offsets, self.feat_dim = k, Fd
        self.num_points = N

    def get_attribute(self, attribute):
        """Activated `scale` (exp), `opacity` (sigmoid), `rot` (normalize); `mlp_*` the module; anything else raw."""
        if attribute in self.activations:
            return self.activations[attribute](getattr(self, "_" + attribute))
        if attribute.startswith("mlp_"):
            return getattr(self, attribute)
        return getattr(self, "_" + attribute)

    def to(self, device):
        super().to(device)
        for name in self._ATTRS:
            v = getattr(self, name)
            if isinstance(v, nn.Parameter):  # registered by an optimizer: move in place, stay a leaf
                v.data = v.data.to(device)
            else:
                setattr(self, name, v.to(device))
        return self

    def requires_grad_(self, flag=True):
        super().requires_grad_(flag)
        for name in self._ATTRS:
            v = getattr(self, name)
            if isinstance(v, nn.Parameter):
                v.requires_grad_(flag)
            else:
                setattr(self, name, v.detach().requires_grad_(flag))
        return self

    def mlps(self):
        return {n: m for n in ("mlp_opacity", "mlp_cov", "mlp_color", "mlp_feature_bank")
                if (m := getattr(self, n)) is not None}


def mix_feature_bank(feat, weights):
    """The reference's multi-resolution feature (scaffold_renderer.py:106-116): feat[:, ::4] and feat[:, ::2] are
    TILED back to F channels (`repeat`), so out[j] = f[4 (j mod F/4)] w0 + f[2 (j mod F/2)] w1 + f[j] w2."""
    return feat[:, ::4].repeat(1, 4) * weights[:, :1] + feat[:, ::2].repeat(1, 2) * weights[:, 1:2] + \
        feat * weights[:, 2:]


def run_mlp(mlp, feat, ob_view, ob_dist):
    """mlp on [feat, view, dist], or [feat, view] when its input width says so."""
    x = torch.cat([feat, ob_view, ob_dist], dim=1)
    return mlp(x if mlp[0].in_features == x.shape[1] else x[:, :-1])


def mlp_outputs(model, vis, camera_center):
    """The three MLP outputs of the visible anchors `vis` (int64) seen from `camera_center`:
    (opacity [Nv,k], color [Nv,3k], cov [Nv,7k])."""
    anchor = model.get_attribute("anchor")[vis]
    feat = model.get_attribute("anchor_feat")[vis]
    ob_view = anchor - camera_center.to(anchor.device)
    ob_dist = ob_view.norm(dim=1, keepdim=True)
    ob_view = ob_view / ob_dist
    if model.use_feat_bank:
        bank = model.mlp_feature_bank
        x = torch.cat([ob_view, ob_dist], dim=1)
        feat = mix_feature_bank(feat, bank(x if bank[0].in_features == 4 else ob_view))
    return (run_mlp(model.mlp_opacity, feat, ob_view, ob_dist), run_mlp(model.mlp_color, feat, ob_view, ob_dist),
            run_mlp(model.mlp_cov, feat, ob_view, ob_dist))


class _ScaffoldDecode(torch.autograd.Function):
    """Compaction and attribute decoding of the neural Gaussians (gsr_scaffold_decode / _backward)."""

    @staticmethod
    def forward(ctx, anchor, offset, scaling, opacity, color, cov, vis, base, M):
        out = _C.scaffold_decode(vis, base, M, anchor, offset, scaling, opacity, color, cov)
        ctx.M = M
        ctx.save_for_backward(vis, base, offset, scaling, opacity, cov)
        return out

    @staticmethod
    def backward(ctx, d_xyz, d_rgb, d_opacity, d_scales, d_rot):
        vis, base, offset, scaling, opacity, cov = ctx.saved_tensors
        g = _C.scaffold_decode_backward(vis, base, ctx.M, offset, scaling, opacity, cov,
                                        (d_xyz, d_rgb, d_opacity, d_scales, d_rot))
        return (*g, None, None, None)


def decode(anchor, offset, scaling, opacity, color, cov, vis):
    """Neural Gaussians of the visible anchors `vis` [Nv] (int64): the reference's rows with opacity > 0, anchor-major
    and offset-minor -> (xyz [M,3], rgb [M,3], opacity [M,1], scales [M,3], rotations [M,4]), differentiable w.r.t.
    anchor [N,3], offset [N,k,3], scaling [N,6] (activated) and the MLP outputs opacity [Nv,k], color [Nv,3k],
    cov [Nv,7k].  One host synchronisation reads the row count M."""
    base, M = _C.scaffold_count(opacity.detach())
    return _ScaffoldDecode.apply(anchor, offset, scaling, opacity.contiguous(), color.contiguous(), cov.contiguous(),
                                 vis, base, M)
