"""The reference's neural-Gaussian decoding (gaustudio/renderers/scaffold_renderer.py:88-159), vectorised in torch.

Run in float64 it is the reference the CUDA decode is checked against; run in float32 it is the torch op sequence the
reference executes (repeat, one [Nv*k, 22] concatenation, boolean-mask gathers), which the end-to-end tests and
tools/scaffold_timing.py put next to the CUDA path.  Differentiable with autograd in either precision."""
import torch
import torch.nn.functional as F


def mix_feature_bank(feat, bank_weight):
    """scaffold_renderer.py:106-116 as written: unsqueeze, strided slices, `repeat` (tiling), squeeze."""
    w = bank_weight.unsqueeze(dim=1)  # [n, 1, 3]
    f = feat.unsqueeze(dim=-1)
    f = f[:, ::4, :1].repeat([1, 4, 1]) * w[:, :, :1] + f[:, ::2, :1].repeat([1, 2, 1]) * w[:, :, 1:2] + \
        f[:, ::1, :1] * w[:, :, 2:]
    return f.squeeze(dim=-1)


def decode(vis, anchor, offset, scaling, opacity, color, cov):
    """vis [Nv] int64; anchor [N,3], offset [N,k,3], scaling [N,6] (activated) full-size; opacity [Nv,k] (the opacity
    MLP's output), color [Nv,3k], cov [Nv,7k] -> (xyz, rgb, opacity, scales, rotations) of the kept rows, and the
    selection mask [Nv*k]."""
    k = offset.shape[1]
    a, grid_offsets, grid_scaling = anchor[vis], offset[vis], scaling[vis]
    Nv = a.shape[0]
    neural_opacity = opacity.reshape([-1, 1])
    mask = (neural_opacity > 0.0).view(-1)
    op = neural_opacity[mask]
    col = color.reshape([Nv * k, 3])
    scale_rot = cov.reshape([Nv * k, 7])
    offs = grid_offsets.reshape([-1, 3])
    cat = torch.cat([grid_scaling, a], dim=-1)
    cat_rep = cat[:, None, :].expand(Nv, k, 9).reshape(Nv * k, 9)  # einops repeat 'n c -> (n k) c'
    masked = torch.cat([cat_rep, col, scale_rot, offs], dim=-1)[mask]
    scaling_repeat, repeat_anchor, col, scale_rot, offs = masked.split([6, 3, 3, 7, 3], dim=-1)
    scales = scaling_repeat[:, 3:] * torch.sigmoid(scale_rot[:, :3])
    rotations = F.normalize(scale_rot[:, 3:7])
    xyz = repeat_anchor + offs * scaling_repeat[:, :3]
    return xyz, col, op, scales, rotations, mask
