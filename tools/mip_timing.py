"""Device time of the Mip-Splatting path on the cfg 3 scene (1M Gaussians, 1920x1080), next to the vanilla path.

    python tools/mip_timing.py [--P 1000000] [--cams 300] [--iters 20] [--out mip_timing.json]

Reports, with the card name and power limit read in the same run:
* ms per view, forward and forward + backward, of `vanilla_renderer` and of `mip_renderer` at kernel_size 0.3 and 0.1
  (CUDA events, mean over --iters after a warm-up), with the binned tile-instance counts that explain the difference;
* per-kernel ms of the projection kernels (k_mip_preprocess_fwd / _bwd next to k_preprocess_fwd / _bwd), from a
  separate torch.profiler run;
* compute_3D_filter for P Gaussians x --cams cameras: the CUDA pass (gsr_mip_filter3d) next to the per-camera torch
  loop of the reference model, written from the same definition."""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gaustudio_b200 import _C, renderers  # noqa: E402
from gaustudio_b200.camera import orbit_cameras  # noqa: E402
from gaustudio_b200.mip import MipPointCloud  # noqa: E402
from gaustudio_b200.synthetic import build_config  # noqa: E402

KERNELS = ("k_preprocess_fwd", "k_preprocess_bwd", "k_mip_preprocess_fwd", "k_mip_preprocess_bwd")


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


def torch_filter3d(xyz, cameras):
    """The reference model's per-camera loop (MipPointCloud.compute_3D_filter), from the definition in include/gsr.h."""
    distance = torch.full((xyz.shape[0],), 100000.0, device=xyz.device)
    valid_points = torch.zeros(xyz.shape[0], device=xyz.device, dtype=torch.bool)
    focal_length = 0.0
    for cam in cameras:
        fx = cam.image_width / (2.0 * math.tan(cam.FoVx * 0.5))
        fy = cam.image_height / (2.0 * math.tan(cam.FoVy * 0.5))
        Rm = torch.tensor(cam.R, device=xyz.device, dtype=torch.float32)
        T = torch.tensor(cam.T, device=xyz.device, dtype=torch.float32)
        p = xyz @ Rm + T[None, :]
        valid_depth = p[:, 2] > 0.2
        z = torch.clamp(p[:, 2], min=0.001)
        x = p[:, 0] / z * fx + cam.image_width / 2.0
        y = p[:, 1] / z * fy + cam.image_height / 2.0
        in_screen = (x >= -0.15 * cam.image_width) & (x <= 1.15 * cam.image_width) & \
                    (y >= -0.15 * cam.image_height) & (y <= 1.15 * cam.image_height)
        valid = valid_depth & in_screen
        distance[valid] = torch.min(distance[valid], z[valid])
        valid_points = valid_points | valid
        focal_length = max(focal_length, fx)
    distance[~valid_points] = distance[valid_points].max()
    return distance / focal_length * (0.2 ** 0.5)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, default=1_000_000)
    ap.add_argument("--cams", type=int, default=300)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mip_timing needs a CUDA device")
    dev = torch.device("cuda")
    base, cams, c = build_config("cfg3", P=a.P, K=1)
    cam = cams[0].to(dev)
    train = orbit_cameras(a.cams, c["radius"], c["elev"], c["W"], c["H"], c["fovx"], c["fovy"])
    model = MipPointCloud.from_model(base).to(dev)
    res = {"card": card(), "P": a.P, "W": c["W"], "H": c["H"], "cameras": a.cams}

    # compute_3D_filter: the CUDA pass against the torch loop (same result up to float32 rounding)
    xyz = model._xyz.detach()
    ours = timed(lambda: _C.mip_filter3d(xyz, train), max(3, a.iters // 4))
    recs = _C.mip_camera_records(train, dev)
    ours_recs = timed(lambda: _C.mip_filter3d(xyz, recs), max(3, a.iters // 4))
    loop = timed(lambda: torch_filter3d(xyz, train), 3)
    f_ours, f_loop = _C.mip_filter3d(xyz, train), torch_filter3d(xyz, train)
    res["filter3d_ms"] = {"cuda_from_cameras": ours, "cuda_from_records": ours_recs, "torch_loop": loop,
                          "max_rel_diff": float(((f_ours - f_loop).abs() / f_loop).max())}
    model.compute_3D_filter(train)

    g = torch.Generator(device=dev).manual_seed(0)
    gimg = torch.randn(3, c["H"], c["W"], device=dev, generator=g)
    res["views"] = {}
    variants = [("vanilla", {"name": "vanilla_renderer"}, base.to(dev)),
                ("mip_k0.3", {"name": "mip_renderer", "kernel_size": 0.3}, model),
                ("mip_k0.1", {"name": "mip_renderer", "kernel_size": 0.1}, model)]
    for name, conf, m in variants:
        r = renderers.make(conf)
        m.requires_grad_(True)

        def fwd():
            with torch.no_grad():
                r.render(cam, m)

        def fwd_bwd():
            out = r.render(cam, m)["render"]
            out.backward(gimg)

        fwd()
        torch.cuda.synchronize()
        res["views"][name] = {"forward_ms": timed(fwd, a.iters), "forward_backward_ms": timed(fwd_bwd, a.iters),
                              "binned_instances": _C.last_num_binned()}
        m.requires_grad_(False)

    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for name, conf, m in variants[:2]:
            r = renderers.make(conf)
            m.requires_grad_(True)
            for _ in range(5):
                r.render(cam, m)["render"].backward(gimg)
            m.requires_grad_(False)
        torch.cuda.synchronize()
    per = {k: 0.0 for k in KERNELS}
    for ev in prof.key_averages():
        for k in KERNELS:
            # "k_preprocess_fwd" is not a substring of "k_mip_preprocess_fwd": the names select one kernel each
            if k in ev.key:
                per[k] += ev.device_time_total / 1000.0 / 5
    res["kernel_ms"] = per
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
