"""Device time of the VisualHull and depth initializers (gaustudio_b200.initializers), median of --reps runs after one
warm-up, CUDA events around each call (each includes the call's own read-backs).  Prints one JSON line per case with
the card's name and power limit read in the same run:
  carve + mesh (visual_hull_carve, then visual_hull_mesh at 0.5) at res 128 and 256 with 100 and 300 cameras of
    1000x750 sphere-silhouette masks, next to a torch restatement on the device of the reference's per-camera
    insideView loop (mask.py:57-68: two insideView calls, a boolean gather and a nonzero per camera; no meshing);
  the depth initializer on 300 views of 1000x750 depth maps (downsampled by 4 as the reference does, host resizes
    and file writes included).
    python tools/hull_timing.py [--reps 3]"""
import argparse, json, math, os, subprocess, sys, tempfile
import numpy as np
import torch
sys.path.insert(0, ".")
sys.path.insert(0, "tests")
from gaustudio_b200 import initializers
from gaustudio_b200.camera import look_at_camera
from gaustudio_b200.synthetic import GaussianPointCloud
import hull_ref64

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=3)
a = ap.parse_args()
dev = torch.device("cuda")
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip().splitlines()[0]
W, H = 1000, 750


def timed(fn, reps=None):
    fn()
    ts = []
    for _ in range(reps or a.reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    return float(np.median(ts))


def report(**kw):
    print(json.dumps({"card": card, **kw}), flush=True)


def cameras(n):
    cams = []
    for k in range(n):
        el = math.radians(25.0 if k % 2 == 0 else -35.0)
        az = 2 * math.pi * k / n
        pos = 4.0 * np.array([math.cos(el) * math.cos(az), math.cos(el) * math.sin(az), math.sin(el)])
        cams.append(look_at_camera(pos, (0.0, 0.0, 0.0), W, H, 0.9, 0.9 * H / W))
    return cams


def sphere_mask(cam, centre=np.array([0.1, -0.2, 0.15]), radius=0.5):
    K = cam.intrinsics.double().numpy()
    u, v = np.meshgrid(np.arange(W) + 0.5, np.arange(H) + 0.5)
    d = np.stack([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], np.ones_like(u)], -1) @ np.asarray(cam.R).T
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    c = -np.asarray(cam.R) @ np.asarray(cam.T)
    dist = np.linalg.norm(centre - c)
    return torch.from_numpy(np.arccos(np.clip(d @ ((centre - c) / dist), -1, 1)) <= math.asin(radius / dist))


all_cams = cameras(300)
for c in all_cams:
    c.mask = sphere_mask(c).to(dev)
r, t = 0.8 * 1.2, np.zeros(3)

for n in (100, 300):
    cams = all_cams[::300 // n][:n]
    for res in (128, 256):
        def run():
            occ = initializers.visual_hull_carve(cams, res, r, t)
            return initializers.visual_hull_mesh(occ, 0.5, r, t)
        ms = timed(run)
        ms_carve = timed(lambda: initializers.visual_hull_carve(cams, res, r, t))
        x = hull_ref64.grid_points(res, r, t, dev)
        specs = [(c.full_proj_transform.to(dev), W, H, c.mask) for c in cams]
        ref_ms = timed(lambda: hull_ref64.carve32(x, specs), reps=1)
        occ = initializers.visual_hull_carve(cams, res, r, t)
        v, f = initializers.visual_hull_mesh(occ, 0.5, r, t)
        differ = int((occ.reshape(-1).bool() != hull_ref64.carve32(x, specs)).sum())
        report(case="visual_hull", cameras=n, mask=f"{W}x{H}", res=res, filled=int(occ.sum()), vertices=v.shape[0],
               faces=f.shape[0], device_ms=ms, carve_ms=ms_carve, torch_restatement_ms=ref_ms,
               nodes_differing_from_float32_loop=differ)
        del x

# ---- depth: 300 views ----
dcams = cameras(300)
u, vv = np.meshgrid(np.arange(W, dtype=np.float32), np.arange(H, dtype=np.float32))
for k, c in enumerate(dcams):
    c.depth = torch.from_numpy(2.0 + 0.5 * np.sin(u / 90.0 + k) * np.cos(vv / 70.0)).float()
    c.image = torch.from_numpy(np.stack([u / W, vv / H, np.full_like(u, 0.5)], -1)).float()
with tempfile.TemporaryDirectory() as ws:
    init = initializers.make({"name": "depth", "workspace_dir": ws})
    ms = timed(lambda: init(GaussianPointCloud.empty(), dcams, overwrite=True))
    m = init(GaussianPointCloud.empty(), dcams, overwrite=True)
    report(case="depth", views=300, size=f"{W}x{H}", gaussians=m._xyz.shape[0], wall_ms=ms,
           note="host PIL resizes, ply / scales.bin writes and reads included")
