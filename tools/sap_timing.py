"""Device time per stage of the Shape-as-Points meshing (extract.mesh_sap) at res 256, sig 2, for a seeded sphere of
100k and 1M oriented points, next to a torch restatement of the reference's DPSR op sequence (scatter_add_ splat,
~15 elementwise spectral ops, gather interpolation; written here from the algorithm, not imported) on the same device.
CUDA events around each stage, median of --reps runs after one warm-up.  The reference meshes with skimage / cumcubes
on the host, which is not timed here.  Prints one JSON line per point count, with the card's name and power limit
read in the same run.
    python tools/sap_timing.py [--reps 10] [--points 100000 1000000]"""
import argparse, json, math, subprocess, sys
import numpy as np
import torch
sys.path.insert(0, ".")
from gaustudio_b200 import _lib, extract

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=10)
ap.add_argument("--points", type=int, nargs="+", default=[100_000, 1_000_000])
ap.add_argument("--res", type=int, default=256)
a = ap.parse_args()
dev, RES, SIG = torch.device("cuda"), a.res, 2.0


def sphere(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(n, 3, generator=g)
    d = d / d.norm(dim=1, keepdim=True)
    return (0.5 * d + torch.tensor([0.1, -0.2, 0.3])).to(dev), d.to(dev)


def ours(xyz, n, t):
    p = torch.empty_like(xyz)
    tr = torch.empty(4, device=dev)
    with t("normalize"), _lib.scratch(dev):
        _lib.call("gsr_sap_normalize", dev, xyz.shape[0], _lib.ptr(xyz), _lib.ALLOC, 1, _lib.ptr(p), _lib.ptr(tr))
    with t("splat"):
        grid = extract._sap_splat(p, n, RES)
    with t("rfftn"):
        spec = torch.fft.rfftn(grid, dim=(1, 2, 3))
    with t("spectral"):
        ph = torch.empty(RES, RES, RES // 2 + 1, dtype=torch.complex64, device=dev)
        _lib.call("gsr_sap_spectral", dev, RES, SIG, _lib.ptr(spec), _lib.ptr(ph))
    with t("irfftn"):
        phi = torch.fft.irfftn(ph, s=(RES,) * 3).contiguous()
    with t("shift_scale"):
        psi = torch.empty_like(phi)
        with _lib.scratch(dev):
            _lib.call("gsr_sap_shift_scale", dev, xyz.shape[0], _lib.ptr(p), RES, _lib.ptr(phi), _lib.ALLOC, 1,
                      _lib.ptr(psi))
    with t("marching_cubes"):  # includes its one blocking count read-back
        v, f = _mc(psi, tr)
    return v, f


def _mc(psi, tr):
    import ctypes as C
    nf = C.c_int64(0)
    with _lib.scratch(dev) as bufs:
        nv = _lib.call("gsr_sap_marching_cubes", dev, RES, _lib.ptr(psi), _lib.ptr(tr), _lib.ALLOC, 1, _lib.ALLOC, 2,
                       _lib.ALLOC, 3, C.byref(nf))
    return nv, nf.value


def _freqs():
    f = torch.tensor(np.fft.fftfreq(RES, d=1.0 / RES), dtype=torch.float32)
    r = torch.tensor(np.fft.rfftfreq(RES, d=1.0 / RES), dtype=torch.float32)
    return torch.stack(torch.meshgrid(f, f, r, indexing="ij"), -1).to(dev)


OMEGA = None
G = None


def _corner_weights(p):
    cs = 1.0 / torch.tensor(float(RES), device=dev)
    i0 = torch.floor(p / cs).long()
    i1 = torch.fmod(torch.ceil(p / cs), RES).long()
    x0, x1 = i0.float() * cs, (i0.float() + 1) * cs
    out = []
    for o in range(8):
        bits = [(o >> 2) & 1, (o >> 1) & 1, o & 1]
        idx = torch.stack([(i1 if b else i0)[:, d] for d, b in enumerate(bits)], 1)
        w = torch.stack([((p[:, d] - x0[:, d]) if b else (p[:, d] - x1[:, d])).abs() / cs for d, b in enumerate(bits)],
                        1).prod(1)
        out.append(((idx[:, 0] * RES + idx[:, 1]) * RES + idx[:, 2], w))
    return out


def torch_reference(xyz, n, t):
    """The reference's op sequence: float32 torch, scatter_add_ splat, per-element spectral ops, gather interpolation."""
    global OMEGA, G
    if OMEGA is None:
        OMEGA = _freqs()
        G = torch.exp(-0.5 * (SIG * 2 * OMEGA.double().norm(dim=-1) / RES) ** 2).float()
    with t("normalize"):
        c = xyz.mean(0)
        s = (xyz - c).abs().max() * 1.2
        p = ((xyz - c) / s + 1.0) / 2.0
    with t("splat"):
        grid = torch.zeros(3, RES ** 3, device=dev)
        for node, w in _corner_weights(p):
            for d in range(3):
                grid[d].scatter_add_(0, node, w * n[:, d])
        grid = grid.view(3, RES, RES, RES)
    with t("rfftn"):
        spec = torch.fft.rfftn(grid, dim=(1, 2, 3))
    with t("spectral"):
        ras = spec.permute(1, 2, 3, 0)[..., None] * G[..., None, None]
        om = OMEGA.unsqueeze(-1) * 2 * np.pi
        r = torch.view_as_real(ras[..., 0])
        ir = torch.stack([-r[..., 1], r[..., 0]], -1)
        div = torch.sum(-ir * om, dim=-2)
        lap = -torch.sum(om ** 2, -2)
        ph = div / (lap + 1e-6)
        ph[0, 0, 0] = 0
        ph = torch.view_as_complex(ph.contiguous())
    with t("irfftn"):
        phi = torch.fft.irfftn(ph, s=(RES,) * 3)
    with t("shift_scale"):
        fv = sum(phi.reshape(-1)[node] * w for node, w in _corner_weights(p))
        phi = phi - fv.mean()
        psi = torch.tanh(-phi / phi[0, 0, 0].abs() * 0.5)
    return psi


class Timer:
    def __init__(self):
        self.ms = {}

    def __call__(self, name):
        timer = self

        class _T:
            def __enter__(self):
                self.e0 = torch.cuda.Event(enable_timing=True); self.e1 = torch.cuda.Event(enable_timing=True)
                self.e0.record()

            def __exit__(self, *exc):
                self.e1.record()
                timer.ms.setdefault(name, []).append((self.e0, self.e1))
        return _T()

    def medians(self):
        torch.cuda.synchronize()
        return {k: float(np.median([a.elapsed_time(b) for a, b in v])) for k, v in self.ms.items()}


q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                   text=True).stdout.strip().splitlines()
card = q[0] if q else torch.cuda.get_device_name(dev)
for N in a.points:
    xyz, n = sphere(N)
    for fn in (ours, torch_reference):
        fn(xyz, n, Timer())  # warm-up: modules, cuFFT plans, allocator
    t_ours, t_ref, total = Timer(), Timer(), []
    for _ in range(a.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        nv, nf = ours(xyz, n, t_ours)
        e1.record()
        torch.cuda.synchronize()
        total.append(e0.elapsed_time(e1))
        torch_reference(xyz, n, t_ref)
    mo, mr = t_ours.medians(), t_ref.medians()
    print(json.dumps({"points": N, "res": RES, "card": card, "mesh_sap_ms": float(np.median(total)),
                      "ours_ms": {k: round(v, 4) for k, v in mo.items()},
                      "torch_reference_ms": {k: round(v, 4) for k, v in mr.items()},
                      "dpsr_ms": {"ours": round(sum(v for k, v in mo.items() if k != "marching_cubes"), 4),
                                  "torch_reference": round(sum(mr.values()), 4)},
                      "vertices": nv, "faces": nf}))
