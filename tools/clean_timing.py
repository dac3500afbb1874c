"""Device time per stage of the point-cloud cleaning (extract.clean_point_cloud) on a seeded sphere of 100k and 1M
oriented surface points, without floaters and with 1 % and 5 % floaters 1000x the scene's size away, next to the host
restatement: scipy's cKDTree (workers=-1) for both passes, and the reference's per-point Python loop of
remove_normal_outliers timed on a subset and reported per point.  CUDA events around each stage (each includes its one count read-back), median of
--reps runs after one warm-up.  Prints one JSON line per scene, with the card's name and power limit read in the same
run.  With --profile, each scene is also run once more under torch.profiler (after the timed runs, so the tracing does
not touch them) and the line gains the device time per kernel of that run.
    python tools/clean_timing.py [--reps 10] [--points 100000 1000000] [--profile 1]"""
import argparse, json, math, subprocess, sys, time
import numpy as np
import torch
sys.path.insert(0, ".")
from gaustudio_b200 import extract

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=10)
ap.add_argument("--points", type=int, nargs="+", default=[100_000, 1_000_000])
ap.add_argument("--host", type=int, default=1, help="also time the host restatement (0: skip)")
ap.add_argument("--profile", type=int, default=0, help="add the device time per kernel of one profiled run")
a = ap.parse_args()
dev = torch.device("cuda")


def scene(n, frac, seed=0):
    g = np.random.default_rng(seed)
    d = g.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    x, nr = 0.5 * d, d
    if frac:
        m = int(round(n * frac))
        x = np.r_[x, g.uniform(-1000, 1000, (m, 3))]
        f = g.normal(size=(m, 3))
        nr = np.r_[nr, f / np.linalg.norm(f, axis=1, keepdims=True)]
    return x.astype(np.float32), nr.astype(np.float32)


def timed(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    out = fn()
    e.record()
    torch.cuda.synchronize()
    return out, s.elapsed_time(e)


def device(x, nr):
    first, t1 = timed(lambda: extract.remove_statistical_outlier(x))
    xs, ns = x[first].contiguous(), nr[first].contiguous()
    second, t2 = timed(lambda: extract.remove_normal_outliers(xs, ns))
    return first[second], t1, t2


def kernels(x, nr):
    """Device time per kernel (ms) of one profiled device(x, nr)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        device(x, nr)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t > 0:
            name = e.key.replace("(anonymous namespace)::", "").split("(")[0].replace("void ", "")
            out[name] = round(out.get(name, 0.0) + t / 1e3, 4)
    return dict(sorted(out.items(), key=lambda kv: -kv[1])[:12])


def host(x, nr):
    from scipy.spatial import cKDTree
    t0 = time.perf_counter()
    d, _ = cKDTree(x).query(x, k=50, workers=-1)
    avg = d.mean(1)
    mean = avg[avg > 0].sum() / len(x)
    std = math.sqrt(((avg[avg > 0] - mean) ** 2).sum() / (len(x) - 1))
    first = np.nonzero((avg > 0) & (avg < mean + 2.0 * std))[0]
    t1 = time.perf_counter()
    xs, ns = x[first], nr[first].astype(np.float64)
    tree = cKDTree(xs)
    _, idx = tree.query(xs, k=20, workers=-1)
    a_ = np.arccos(np.minimum(np.abs(np.einsum("ijk,ik->ij", ns[idx[:, 1:]], ns)), 1.0))
    keep = a_.mean(1) < math.pi / 4
    t2 = time.perf_counter()
    sub = min(2000, len(xs))  # the reference's loop, one KDTree query per point
    t3 = time.perf_counter()
    for i in range(sub):
        _, ii = tree.query(xs[i], k=20)
        np.mean(np.arccos(np.abs(np.dot(ns[ii[1:]], ns[i]))))
    t4 = time.perf_counter()
    return first[keep], (t1 - t0) * 1e3, (t2 - t1) * 1e3, (t4 - t3) / sub * 1e6


q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                   text=True).stdout.strip().splitlines()
card = q[0] if q else torch.cuda.get_device_name(dev)
for N in a.points:
    for frac in (0.0, 0.01, 0.05):
        xn, nn = scene(N, frac)
        x, nr = torch.from_numpy(xn).to(dev), torch.from_numpy(nn).to(dev)
        device(x, nr)  # warm-up
        runs = [device(x, nr) for _ in range(a.reps)]
        t1 = float(np.median([r[1] for r in runs]))
        t2 = float(np.median([r[2] for r in runs]))
        out = {"points": int(len(xn)), "floaters": frac, "card": card, "kept": int(runs[0][0].numel()),
               "statistical_ms": t1, "normal_ms": t2, "clean_ms": t1 + t2}
        if a.profile:
            out["kernel_ms"] = kernels(x, nr)
        if a.host:
            keep_h, h1, h2, loop_us = host(xn, nn)
            out.update(host_ckdtree_statistical_ms=h1, host_ckdtree_normal_ms=h2, host_loop_us_per_point=loop_us,
                       host_kept=int(len(keep_h)))
        print(json.dumps(out), flush=True)
