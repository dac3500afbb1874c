"""Contribution statistics and pruning on cfg3 (1M Gaussians, 1920x1080, 200 orbit views):

  * device ms of one statistics pass (gsr_contribution) next to the compositing forward (k_render_fwd, the library's
    per-stage events) on the same view;
  * the whole prune.contribution over all views (forward + pass per view, host clock around a synchronised run);
  * the fraction of Gaussians with count == 0 over all views;
  * forward and forward + backward ms per view before pruning, after the count == 0 prune and after ratio 0.66;
  * PSNR of the pruned renders against the unpruned ones.

cfg3 is a random ball: its pruning fractions and PSNRs say nothing about trained scenes.

    python tools/prune_timing.py [--views 200] [--timed 20] [--out prune_timing.json]

The card name and power limit are read in the same run."""
import argparse
import ctypes
import json
import math
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gaustudio_b200 import _C, _lib, renderers  # noqa: E402
from gaustudio_b200 import prune as PR  # noqa: E402
from gaustudio_b200.synthetic import GaussianPointCloud, build_config  # noqa: E402

DEV = torch.device("cuda:0")
RENDER_FWD = 4  # stage index of k_render_fwd in gsr_profile_read


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name() + ", power limit unknown"


def events_ms(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def pass_vs_forward(model, cam, r, iters):
    L = _lib.lib()
    with torch.no_grad():
        out, H, W = PR._forward(r, cam, model)
    P = model._xyz.shape[0]
    acc = (torch.zeros(P, dtype=torch.float64, device=DEV), torch.zeros(P, dtype=torch.int64, device=DEV),
           torch.zeros(P, dtype=torch.float32, device=DEV))
    pass_ms = events_ms(lambda: _C.contribution(P, H, W, out[6], out[0], out[7], out[8], *acc), iters)
    with torch.no_grad():
        PR._forward(r, cam, model)
        torch.cuda.synchronize()
        L.gsr_profile_enable(1)
        for _ in range(iters):
            PR._forward(r, cam, model)
        torch.cuda.synchronize()
        ms, cn = (ctypes.c_float * 8)(), (ctypes.c_int * 8)()
        L.gsr_profile_read(ms, cn)
        L.gsr_profile_enable(0)
    return pass_ms, ms[RENDER_FWD] / max(cn[RENDER_FWD], 1)


def step_ms(model, cams, r, iters):
    """(forward ms, forward + backward ms) per view over the first `iters` cameras."""
    def fwd():
        with torch.no_grad():
            for c in cams[:iters]:
                r.render(c, model)

    def fwd_bwd():
        for c in cams[:iters]:
            o = r.render(c, model)
            (o["render"].sum() + o["rendered_depth"].sum()).backward()
    model.requires_grad_(True)
    f = events_ms(fwd, 1) / iters
    fb = events_ms(fwd_bwd, 1) / iters
    model.requires_grad_(False)
    return f, fb


def renders(model, cams, r):
    with torch.no_grad():
        return [r.render(c, model)["render"].clamp(0, 1) for c in cams]


def psnr(a, b):
    mse = sum(float(((x - y) ** 2).mean()) for x, y in zip(a, b)) / len(a)
    return float("inf") if mse == 0 else 10 * math.log10(1.0 / mse)


def clone(model):
    return GaussianPointCloud(*[getattr(model, k).detach().clone() for k in PR.ATTRS], model.max_sh_degree,
                              model.active_sh_degree)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=200)
    ap.add_argument("--timed", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    model, cams, cfg = build_config("cfg3", K=a.views)
    model.active_sh_degree = 3
    model.to(DEV)
    cams = [c.to(DEV) for c in cams]
    r = renderers.make("vanilla_renderer")
    res = {"card": card(), "config": "cfg3", "P": model._xyz.shape[0], "views": len(cams),
           "note": "cfg3 is a random ball: pruning fractions and PSNRs say nothing about trained scenes"}
    res["pass_ms"], res["render_fwd_ms"] = pass_vs_forward(model, cams[0], r, 20)
    PR.contribution(model, cams[:2], r)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    c = PR.contribution(model, cams, r)
    torch.cuda.synchronize()
    res["contribution_all_views_s"] = time.perf_counter() - t0
    P = res["P"]
    zero = c["count"] == 0
    res["count_zero_fraction"] = float(zero.sum()) / P
    ref = renders(model, cams, r)
    res["before"] = dict(zip(("fwd_ms", "fwd_bwd_ms"), step_ms(model, cams, r, a.timed)))
    m0 = clone(model)
    PR.prune(m0, ~zero)
    res["after_count_zero"] = dict(zip(("fwd_ms", "fwd_bwd_ms"), step_ms(m0, cams, r, a.timed)), P=m0._xyz.shape[0],
                                   psnr_db=psnr(renders(m0, cams, r), ref))
    del m0
    m1 = clone(model)
    PR.prune(m1, PR.select(PR.significance(model, c), 0.66))
    res["after_ratio_0.66"] = dict(zip(("fwd_ms", "fwd_bwd_ms"), step_ms(m1, cams, r, a.timed)), P=m1._xyz.shape[0],
                                   psnr_db=psnr(renders(m1, cams, r), ref))
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
