"""Contribution-based pruning: how much each Gaussian adds to a set of views, a significance score built on it, and an
order-preserving prune.  The first step of 3DGS post-processing (the reference's planned `gs-compress`); DESIGN.md §7l
has the contract.

    contrib = contribution(model, cameras, renderer)     # one forward + one statistics pass per view
    keep = contrib["count"] > 0                           # drop what no view ever depended on, or
    keep = select(significance(model, contrib), 0.66)     # keep the 34 % most significant
    prune(model, keep, optimizer)

The statistics come from the forward's own blend decisions (`gsr_contribution`), so a Gaussian with `count == 0` over
a set of views can be removed without changing a single bit of those views' renders.
"""
import math

import torch

from . import _C
from .densify import ATTRS, _is_optimised, _replace, _state_of, _torch_optimizer
from .rasterizer import check_exactly_one_of
from .renderers.mip_renderer import MipRenderer

_STATS = ("xyz_gradient_accum", "denom", "max_radii2D")


def _refuse_renderer(renderer):
    from .renderers.scaffold_renderer import ScaffoldRenderer
    from .renderers.surfel_renderer import SurfelRenderer
    if isinstance(renderer, SurfelRenderer):
        raise NotImplementedError("contribution: the surfel (2DGS) compositing has no statistics pass")
    if isinstance(renderer, ScaffoldRenderer):
        raise NotImplementedError("contribution: Scaffold-GS decodes its Gaussians per view; they have no persistent "
                                  "rows to score")


def _forward(renderer, camera, model):
    """The renderer's forward of one view through the _C call its render() makes -> (the 9-tuple of
    _C.rasterize_gaussians, H, W)."""
    can_fuse = getattr(renderer, "_can_fuse", None)
    if can_fuse is not None and can_fuse(model):  # vanilla_renderer with fused_activations
        m = model
        P = m._xyz.shape[0]
        rs = renderer.raster_settings(camera, m.active_sh_degree)
        e = torch.Tensor([])
        out = _C.rasterize_gaussians(rs.bg, m._xyz.detach(), e, m._opacity.detach(), m._scale.detach(),
                                     m._rot.detach(), rs.scale_modifier, e, rs.viewmatrix, rs.projmatrix, rs.tanfovx,
                                     rs.tanfovy, rs.image_height, rs.image_width, e, rs.sh_degree, rs.campos,
                                     rs.prefiltered, rs.debug,
                                     _fused=(m._f_dc.detach().reshape(P, -1, 3), m._f_rest.detach().reshape(P, -1, 3)))
    else:
        xyz, shs, colors, opacity, scales, rotations, cov3D = renderer.get_gaussians_properties(camera, model)
        check_exactly_one_of(shs, colors, scales, rotations, cov3D)
        degree = model.active_sh_degree if shs is not None else 1
        rs = renderer.raster_settings(camera, degree)
        e = torch.Tensor([])
        opt = lambda t: e if t is None else t
        args = (rs.bg, xyz, opt(colors), opacity, opt(scales), opt(rotations), rs.scale_modifier, opt(cov3D),
                rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, rs.image_height, rs.image_width, opt(shs),
                rs.sh_degree, rs.campos, rs.prefiltered, rs.debug)
        if hasattr(rs, "kernel_size"):
            out = _C.rasterize_gaussians_mip(*args, rs.kernel_size)
        else:
            out = _C.rasterize_gaussians(*args)
    return out, int(rs.image_height), int(rs.image_width)


@torch.no_grad()
def contribution(model, cameras, renderer):
    """Per-Gaussian statistics of the blend weights w = alpha T the forward composites, over `cameras`, rendered with
    `renderer`'s own settings and attribute gathering (vanilla_renderer, fused or not, and mip_renderer).

    Returns dict(weight=float64[P]: sum of w over every pixel of every view; count=int64[P]: the pixels at which the
    forward's walk reached the transmittance test for the Gaussian, i.e. the pixels it blended plus the pixels it ended
    (T (1 - alpha) < 1e-4, no weight), so count == 0 means no view depended on it; max_weight=float32[P]: the largest w;
    views=len(cameras)).  The pass adds no host synchronisation to the forward's own.  surfel_renderer and
    scaffold_renderer raise NotImplementedError."""
    _refuse_renderer(renderer)
    cameras = list(cameras)
    if not cameras:
        raise ValueError("contribution: no cameras")
    if isinstance(renderer, MipRenderer) and getattr(model, "filter_3D", None) is None:
        raise ValueError("mip_renderer needs a model with filter_3D: call compute_3D_filter(cameras) on a MipPointCloud")
    dev = model._xyz.device
    if dev.type != "cuda":
        raise RuntimeError("contribution runs on CUDA (sm_90a) only: move the model to a CUDA device")
    P = model._xyz.shape[0]
    weight = torch.zeros(P, dtype=torch.float64, device=dev)
    count = torch.zeros(P, dtype=torch.int64, device=dev)
    max_weight = torch.zeros(P, dtype=torch.float32, device=dev)
    for cam in cameras:
        out, H, W = _forward(renderer, cam, model)
        if P:
            _C.contribution(P, H, W, out[6], out[0], out[7], out[8], weight, count, max_weight)
    return dict(weight=weight, count=count, max_weight=max_weight, views=len(cameras))


def _volume(model):
    """Product of the three activated scales the renderers use: the 3D-filtered ones for a model with a filter_3D."""
    if getattr(model, "filter_3D", None) is not None:
        s = model.get_scaling_with_3D_filter
    else:
        s = model.get_attribute("scale")
    return torch.prod(s.detach().to(torch.float64), dim=-1)


@torch.no_grad()
def significance(model, contrib, v_pow=0.1):
    """LightGaussian's volume-weighted global significance, with the blend weight as the hit measure:

        score_i = weight_i * (V_i / V_ref) ** v_pow,

    V_i the product of Gaussian i's three activated scales (the 3D-filtered scales for a Mip model), V_ref the volume at
    position floor(0.9 P) of the volumes sorted in descending order.  float64 [P].  The formula follows the LightGaussian
    paper; bit parity with its code is not claimed."""
    w = contrib["weight"]
    P = model._xyz.shape[0]
    if tuple(w.shape) != (P,):
        raise ValueError(f"significance: the statistics have {tuple(w.shape)} rows, the model has {P} Gaussians")
    if P == 0:
        return torch.zeros(0, dtype=torch.float64, device=w.device)
    V = _volume(model).to(w.device)
    v_ref = torch.sort(V, descending=True).values[int(math.floor(0.9 * P))]
    return w.to(torch.float64) * torch.pow(V / v_ref, float(v_pow))


def select(score, prune_ratio):
    """Keep mask [P] of the P - floor(prune_ratio P) highest scores; ties go to the lower index (a stable sort), so the
    count is exact."""
    r = float(prune_ratio)
    if not 0.0 <= r <= 1.0:
        raise ValueError(f"select: prune_ratio must be in [0, 1], got {prune_ratio!r}")
    P = score.shape[0]
    n_keep = P - int(math.floor(r * P))
    order = torch.sort(score, descending=True, stable=True).indices
    keep = torch.zeros(P, dtype=torch.bool, device=score.device)
    keep[order[:n_keep]] = True
    return keep


@torch.no_grad()
def prune(model, keep, optimizer=None):
    """Order-preserving compaction to the rows where `keep` (bool [P]) is True: the six attributes, a Mip model's
    filter_3D, the densification statistics when present, and the optimizer state (FusedAdam, torch.optim or the plugin
    BaseOptimizer; every state tensor shaped like its parameter is compacted, `step` is kept).

    Like densify.densify_and_prune it replaces the model's attribute tensors: rebuild any `parallel.GradBucket` and
    `graphs.GraphedViewStep` made before.  Returns dict(P_before, P_after, pruned)."""
    from .scaffold import ScaffoldPointCloud
    if isinstance(model, ScaffoldPointCloud):
        raise NotImplementedError("prune: a ScaffoldPointCloud has anchors, not Gaussians")
    for a in ATTRS:
        if not hasattr(model, a):
            raise TypeError(f"prune: the model has no {a} (a 3DGS point cloud is needed)")
    P = model._xyz.shape[0]
    if keep.dtype != torch.bool or tuple(keep.shape) != (P,):
        raise ValueError(f"prune: keep must be a bool tensor of shape ({P},), got {keep.dtype} {tuple(keep.shape)}")
    dev = model._xyz.device
    idx = keep.to(dev).nonzero().squeeze(1)
    opt = _torch_optimizer(optimizer)
    for a in ATTRS:
        old = getattr(model, a)
        st = _state_of(opt, old) if _is_optimised(opt, old) else None
        new_state = None
        if st is not None:
            new_state = {k: (v[idx].contiguous() if torch.is_tensor(v) and v.shape == old.shape else v)
                         for k, v in st.items()}
        _replace(model, opt, a, old, old.detach()[idx].contiguous(), new_state)
    if getattr(model, "filter_3D", None) is not None:
        model.filter_3D = model.filter_3D[idx].contiguous()
    for name in _STATS:
        t = getattr(model, name, None)
        if t is not None:
            setattr(model, name, t[idx.to(t.device)].contiguous())
    n = int(idx.numel())
    if hasattr(model, "num_points"):
        model.num_points = n
    return dict(P_before=P, P_after=n, pruned=P - n)
