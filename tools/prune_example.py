"""Post-processing: prune a trained 3DGS checkpoint by how much each Gaussian contributes to its training views.

    python tools/prune_example.py point_cloud.ply cameras.json pruned.ply [--ratio 0.66] [--sh-degree 3]
                                  [--renderer vanilla_renderer] [--kernel-size 0.1]

Renders every camera of cameras.json once, accumulates the blend-weight statistics of gaustudio_b200.prune, and
writes the model without its least significant Gaussians.  --ratio r drops floor(r P) Gaussians by LightGaussian's
volume-weighted significance; --ratio 0 drops only the Gaussians no view depended on (count == 0), which leaves every
training view's render bit-identical.  A Mip-Splatting checkpoint (a PLY with filter_3D) is rendered with mip_renderer
whatever --renderer says."""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gaustudio_b200 import io, renderers  # noqa: E402
from gaustudio_b200 import prune as PR  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("ply")
    ap.add_argument("cameras")
    ap.add_argument("out")
    ap.add_argument("--ratio", type=float, default=0.66)
    ap.add_argument("--sh-degree", type=int, default=3)
    ap.add_argument("--renderer", default="vanilla_renderer")
    ap.add_argument("--kernel-size", type=float, default=0.1)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    model = io.load_ply(a.ply, sh_degree=a.sh_degree, active_sh_degree=a.sh_degree, device=dev)
    cams = [c.to(dev) for c in io.load_cameras_json(a.cameras)]
    if getattr(model, "filter_3D", None) is not None:
        r = renderers.make({"name": "mip_renderer", "kernel_size": a.kernel_size})
    else:
        r = renderers.make(a.renderer)
    c = PR.contribution(model, cams, r)
    keep = c["count"] > 0 if a.ratio == 0 else PR.select(PR.significance(model, c), a.ratio)
    res = PR.prune(model, keep)
    io.export_ply(model, a.out)
    print(f"{len(cams)} views; {int((c['count'] == 0).sum())} of {res['P_before']} Gaussians never reached; "
          f"kept {res['P_after']} -> {a.out}")


if __name__ == "__main__":
    main()
