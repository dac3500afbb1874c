"""Seeded Scaffold-GS fixtures.

decode_case: the inputs of the neural-Gaussian decoding alone, with anchors whose offsets all, none or some survive
(opacity exactly 0 included, which is dropped), rotations that hit the 1e-12 normalisation clamp and zero scalings.
model: a ScaffoldPointCloud in front of a camera, with anchors behind the near plane and off screen, tiny scales, and
MLP weights drawn so that about half of the offsets survive."""
import math

import torch

W, H = 160, 120


def decode_case(N, k, seed, frac=0.6):
    g = torch.Generator().manual_seed(seed)
    vis = torch.nonzero(torch.rand(N, generator=g) < frac).flatten()
    Nv = vis.numel()
    anchor = torch.randn(N, 3, generator=g)
    offset = torch.randn(N, k, 3, generator=g)
    scaling = torch.exp(torch.randn(N, 6, generator=g) * 0.5 - 2.0)
    scaling[::13] = 0.0  # degenerate: offsets and scales collapse
    opacity = torch.tanh(torch.randn(Nv, k, generator=g))
    if Nv > 3:
        opacity[0] = opacity[0].abs() + 0.01      # every offset survives
        opacity[1] = -opacity[1].abs()            # none survives
        opacity[2, ::2] = 0.0                     # exactly 0: dropped
    color = torch.sigmoid(torch.randn(Nv, 3 * k, generator=g))
    cov = torch.randn(Nv, 7 * k, generator=g)
    c = cov.view(Nv, k, 7)
    c[::5, 0, 3:7] = 0.0     # |q| = 0: the clamp holds the norm at 1e-12
    c[1::5, -1, 3:7] = 1e-14  # |q| = 2e-14 < 1e-12: clamped as well
    return dict(vis=vis, anchor=anchor, offset=offset, scaling=scaling, opacity=opacity, color=color, cov=cov)


def camera(W=W, H=H, device="cpu"):
    from gaustudio_b200.camera import look_at_camera
    fovy = math.radians(50.0)
    fovx = 2 * math.atan(math.tan(fovy / 2) * W / H)
    return look_at_camera((0.0, -3.0, 1.0), (0.0, 0.0, 0.0), W, H, fovx, fovy).to(device)


def model(N, k, F=32, seed=0, use_feat_bank=False, use_dist=True, radius=1.0, shell=False, outliers=True,
          device="cpu"):
    """Anchors uniform in a ball (or on a sphere with shell=True); with `outliers`, 4 % behind the camera and 4 % far
    off screen."""
    from gaustudio_b200.scaffold import ScaffoldPointCloud, make_mlps
    ga = torch.Generator().manual_seed(seed)  # positions
    d = torch.randn(N, 3, generator=ga)
    d = d / d.norm(dim=1, keepdim=True)
    anchor = radius * d * (1.0 if shell else torch.rand(N, 1, generator=ga) ** (1 / 3))
    g = torch.Generator().manual_seed(seed)   # everything else
    n_out = N // 25 if outliers else 0
    if n_out:
        anchor[:n_out] = torch.tensor([0.0, -3.0, 1.0]) + 0.3 * torch.randn(n_out, 3, generator=g) + \
            torch.tensor([0.0, -1.5, 0.5])                       # behind the camera
        anchor[n_out:2 * n_out] = torch.randn(n_out, 3, generator=g) + torch.tensor([40.0, 0.0, 0.0])  # off screen
    offset = 0.5 * torch.randn(N, k, 3, generator=g)
    feat = torch.randn(N, F, generator=g)
    opacity = torch.zeros(N, 1)
    scale = torch.cat([math.log(0.04) + 0.2 * torch.randn(N, 3, generator=g),
                       math.log(0.03) + 0.2 * torch.randn(N, 3, generator=g)], 1)
    if outliers:
        scale[2 * n_out:2 * n_out + 3] = -30.0  # degenerate: exp(-30)
    rot = torch.randn(N, 4, generator=g)
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(seed + 1)
        mlps = make_mlps(F, k, use_feat_bank, use_dist)
        with torch.no_grad():
            mlps["mlp_opacity"][2].bias.zero_()  # tanh(x) > 0 iff x > 0: about half of the offsets survive
            mlps["mlp_opacity"][2].weight.mul_(3.0)
    m = ScaffoldPointCloud(anchor, offset, feat, opacity, scale, rot, **mlps)
    return m.to(device)

