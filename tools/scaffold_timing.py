"""Device time of the Scaffold-GS path per view: anchor visibility, the anchor MLPs, the neural-Gaussian decoding
(forward and backward) and the Mip rasterizer (forward and backward), at 100k and 300k anchors, k = 10, 1920x1080.

    python tools/scaffold_timing.py [--anchors 100000 300000] [--iters 20] [--out scaffold_timing.json]

Reports, with the card name and power limit read in the same run, the mean ms per call over --iters after a warm-up
(CUDA events; the decode's count read is a host synchronisation and is inside its time), and the CUDA decode next to
the torch restatement of the reference's op sequence (tests/scaffold_ref64.py run in float32), forward and forward +
backward."""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import scaffold_ref64 as SR  # noqa: E402
from gaustudio_b200 import _C, renderers, scaffold  # noqa: E402
from gaustudio_b200.camera import look_at_camera  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name() + ", power limit unknown"


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def scene(N, k, F, seed=0):
    """Anchors in a ball of radius 1 seen from 3 units away; about half of the offsets survive."""
    from gaustudio_b200.scaffold import ScaffoldPointCloud, make_mlps
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(N, 3, generator=g)
    anchor = d / d.norm(dim=1, keepdim=True) * torch.rand(N, 1, generator=g) ** (1 / 3)
    scale = torch.cat([math.log(0.01) + 0.2 * torch.randn(N, 3, generator=g),
                       math.log(0.005) + 0.2 * torch.randn(N, 3, generator=g)], 1)
    torch.manual_seed(seed)
    mlps = make_mlps(F, k)
    with torch.no_grad():
        mlps["mlp_opacity"][2].bias.zero_()
    return ScaffoldPointCloud(anchor, 0.5 * torch.randn(N, k, 3, generator=g), torch.randn(N, F, generator=g),
                              torch.zeros(N, 1), scale, torch.randn(N, 4, generator=g), **mlps).to("cuda")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--anchors", type=int, nargs="+", default=[100_000, 300_000])
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--feat", type=int, default=32)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    W, H = 1920, 1080
    fovy = math.radians(49.1)
    cam = look_at_camera((0.0, -3.0, 1.0), (0.0, 0.0, 0.0), W, H, 2 * math.atan(math.tan(fovy / 2) * W / H),
                         fovy).to("cuda")
    r = renderers.make("scaffold_renderer")
    res = {"card": card(), "W": W, "H": H, "k": args.k, "feat_dim": args.feat, "iters": args.iters, "runs": []}
    for N in args.anchors:
        m = scene(N, args.k, args.feat).requires_grad_(True)
        visible = r.prefilter_voxel(cam, m)
        vis = visible.nonzero().flatten()
        o, c, s = scaffold.mlp_outputs(m, vis, cam.camera_center)
        anchor, offset, scaling = m.get_attribute("anchor"), m.get_attribute("offset"), m.get_attribute("scale")
        out = scaffold.decode(anchor, offset, scaling, o, c, s, vis)
        M = out[0].shape[0]
        base, _ = _C.scaffold_count(o.detach())
        ups = [torch.randn_like(t) for t in out]
        leaves = [t.detach().requires_grad_(True) for t in (anchor, offset, scaling, o, c, s)]
        props = (out[0].detach(), None, out[1].detach(), out[2].detach(), out[3].detach(), out[4].detach(), None)
        w = torch.randn(3, H, W, device="cuda")

        def torch_decode():
            return SR.decode(vis, *[t.detach() for t in (anchor, offset, scaling, o, c, s)])[:5]

        def torch_decode_fb():
            y = SR.decode(vis, *leaves)[:5]
            torch.autograd.backward(y, ups)

        def cuda_decode_fb():
            y = scaffold.decode(*leaves[:3], *leaves[3:], vis)
            torch.autograd.backward(y, ups)

        def raster_fb():
            p = tuple(t.detach().requires_grad_(True) if t is not None else None for t in props)
            (img, *_), _ = r.rasterize(cam, m, p)
            (img * w).sum().backward()

        def render_fb():
            (r.render(cam, m)["render"] * w).sum().backward()

        with torch.no_grad():
            t = dict(
                visibility=timed(lambda: r.prefilter_voxel(cam, m), args.iters),
                decode_fwd=timed(lambda: scaffold.decode(anchor, offset, scaling, o, c, s, vis), args.iters),
                decode_bwd=timed(lambda: _C.scaffold_decode_backward(vis, base, M, offset, scaling, o, s, ups),
                                 args.iters),
                raster_fwd=timed(lambda: r.rasterize(cam, m, props), args.iters),
                torch_decode_fwd=timed(torch_decode, args.iters),
                render_fwd=timed(lambda: r.render(cam, m), args.iters))
        t["mlps_fwd"] = timed(lambda: scaffold.mlp_outputs(m, vis, cam.camera_center), args.iters)
        t["decode_fwd_bwd"] = timed(cuda_decode_fb, args.iters)
        t["torch_decode_fwd_bwd"] = timed(torch_decode_fb, args.iters)
        t["raster_fwd_bwd"] = timed(raster_fb, args.iters)
        t["render_fwd_bwd"] = timed(render_fb, args.iters)
        run = {"anchors": N, "visible": int(vis.numel()), "neural_gaussians": M, "ms": {k: round(v, 4) for k, v in t.items()}}
        res["runs"].append(run)
        print(json.dumps(run), flush=True)
    print(json.dumps({"card": res["card"]}))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
