"""Device time of the Gaussian initializers (gaustudio_b200.initializers), median of --reps runs after one warm-up,
CUDA events around each call (each includes the call's own read-backs).  Prints one JSON line per case with the
card's name and power limit read in the same run:
  dist2 at 100k and 1M surface points, without floaters and with 1 % far floaters (1000x the scene away), next to
    scipy's cKDTree (workers=-1, k=4) on the host;
  the mesh initializer at n = 3 on a UV sphere of >= 1M faces, next to a torch restatement of the reference's
    MeshInitializer.build_model ops on the device (its vertex normals taken as given);
  the voxel initializer at voxel_size 1/256 and 1/512 on that sphere and on one triangle spanning the grid.
    python tools/init_timing.py [--reps 5]"""
import argparse, json, subprocess, sys, time
import numpy as np
import torch
sys.path.insert(0, ".")
from gaustudio_b200 import initializers
from gaustudio_b200.synthetic import GaussianPointCloud

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=5)
a = ap.parse_args()
dev = torch.device("cuda")
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip().splitlines()[0]


def timed(fn):
    fn()
    ts = []
    for _ in range(a.reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    return float(np.median(ts))


def report(**kw):
    print(json.dumps({"card": card, **kw}), flush=True)


def cloud(n, frac, seed=0):
    g = np.random.default_rng(seed)
    d = g.normal(size=(n, 3))
    x = 0.5 * d / np.linalg.norm(d, axis=1, keepdims=True)
    m = int(round(n * frac))
    if m:
        x = np.r_[x, g.uniform(-500, 500, (m, 3))]
    return x.astype(np.float32)


def uv_sphere(n_lat, n_lon):
    th = np.linspace(0, np.pi, n_lat + 1)[1:-1]
    ph = np.linspace(0, 2 * np.pi, n_lon, endpoint=False)
    T, P = np.meshgrid(th, ph, indexing="ij")
    v = np.stack([np.sin(T) * np.cos(P), np.sin(T) * np.sin(P), np.cos(T)], -1).reshape(-1, 3)
    v = np.concatenate([[[0, 0, 1]], v, [[0, 0, -1]]]) * 0.5
    i = np.arange(n_lat - 2)[:, None]
    j = np.arange(n_lon)[None, :]
    idx = lambda i, j: 1 + i * n_lon + j % n_lon
    quads = [np.stack([idx(i, j), idx(i + 1, j), idx(i + 1, j + 1)], -1),
             np.stack([idx(i, j), idx(i + 1, j + 1), idx(i, j + 1)], -1)]
    jj = np.arange(n_lon)
    caps = [np.stack([np.zeros(n_lon, int), idx(0, jj), idx(0, jj + 1)], -1),
            np.stack([np.full(n_lon, len(v) - 1), idx(n_lat - 2, jj + 1), idx(n_lat - 2, jj)], -1)]
    f = np.concatenate([q.reshape(-1, 3) for q in quads] + caps)
    col = 0.5 + 0.5 * np.sin(3 * v)
    return (torch.from_numpy(v.astype(np.float32)).to(dev), torch.from_numpy(f.astype(np.int64)).to(dev),
            torch.from_numpy(col.astype(np.float32)).to(dev))


# ---- dist2 ----
from scipy.spatial import cKDTree
for n in (100_000, 1_000_000):
    for frac in (0.0, 0.01):
        x = cloud(n, frac)
        xd = torch.from_numpy(x).to(dev)
        ms = timed(lambda: initializers.dist2(xd))
        t0 = time.perf_counter()
        cKDTree(x).query(x, k=4, workers=-1)
        host = (time.perf_counter() - t0) * 1e3
        report(case="dist2", points=len(x), floaters=frac, device_ms=ms, ckdtree_host_ms=host)

# ---- mesh ----
v, f, col = uv_sphere(708, 708)  # 1,000,536 faces
F = f.shape[0]
init = initializers.make({"name": "mesh", "n_gaussians_per_surface_triangle": 3})
model = GaussianPointCloud.empty(sh_degree=1)
ms = timed(lambda: init(model, (v, f, col)))
vn = initializers.vertex_normals(v, f)
B = torch.tensor([[1 / 2, 1 / 4, 1 / 4], [1 / 4, 1 / 2, 1 / 4], [1 / 4, 1 / 4, 1 / 2]], device=dev)[..., None]
rad = 1. / 2. / (np.sqrt(3.) + 1.)


def torch_ref():
    """MeshInitializer.build_model's torch ops (mesh.py:212-250) + normal2rotation + create_from_attribute's RGB2SH."""
    fv, fn_, fc = v[f], vn[f], col[f]
    pts = (fv[:, None] * B[None]).sum(-2).reshape(-1, 3)
    nr = torch.nn.functional.normalize((fn_[:, None] * B[None]).sum(-2).reshape(-1, 3), dim=-1)
    q = _n2r(nr)
    c = ((fc[:, None] * B[None]).sum(-2).reshape(-1, 3) - 0.5) / 0.28209479177387814
    e = (fv - fv[:, [1, 2, 0]]).norm(dim=-1).min(dim=-1)[0] * rad
    s = e.clamp_min(0.).reshape(F, -1, 1).expand(-1, 3, 2).clone().reshape(-1, 2)
    s = torch.log(torch.cat([s, torch.zeros(s.shape[0], 1, device=dev)], -1) * 2 + 1e-7)
    return pts, q, c, s


def _n2r(n):
    n = torch.nn.functional.normalize(n)
    w0 = torch.tensor([[1, 0, 0]], device=dev).expand(n.shape)
    R0 = w0 - torch.sum(w0 * n, -1, True) * n
    R0 *= torch.sign(R0[:, :1])
    R0 = torch.nn.functional.normalize(R0)
    R1 = torch.cross(n, R0, dim=-1)
    R1 *= torch.sign(R1[:, 1:2]) * torch.sign(n[:, 2:])
    R = torch.stack([R0, R1, n], -1)
    tr = R[:, 0, 0] + R[:, 1, 1] + R[:, 2, 2] + 1e-6
    r = torch.sqrt(1 + tr) / 2
    return torch.stack([r, (R[:, 2, 1] - R[:, 1, 2]) / (4 * r), (R[:, 0, 2] - R[:, 2, 0]) / (4 * r),
                        (R[:, 1, 0] - R[:, 0, 1]) / (4 * r)], -1)


ref_ms = timed(torch_ref)
report(case="mesh", n=3, faces=F, gaussians=3 * F, device_ms=ms, torch_restatement_ms=ref_ms,
       note="device_ms includes the vertex normals and the index check's read-back")

# ---- voxel ----
span = (torch.tensor([[-1, -1, -1], [1, 1, -0.2], [-0.3, 1, 1]], device=dev),
        torch.tensor([[0, 1, 2]], device=dev), torch.eye(3, device=dev))
for name, mesh in (("sphere", (v, f, col)), ("spanning_triangle", span)):
    for vs in (1 / 256, 1 / 512):
        vinit = initializers.make({"name": "voxel", "voxel_size": vs})
        gen = torch.Generator().manual_seed(0)
        ms = timed(lambda: vinit(GaussianPointCloud.empty(sh_degree=0), mesh, generator=gen))
        vn_, _, _ = initializers.normalize_mesh(mesh[0])
        cells, off, tris = initializers.voxelize(vn_, mesh[1], vinit.res, vs)
        ms_vox = timed(lambda: initializers.voxelize(vn_, mesh[1], vinit.res, vs))
        report(case="voxel", mesh=name, faces=int(mesh[1].shape[0]), voxel_size=vs, occupied=int(cells.shape[0]),
               pairs=int(tris.shape[0]), device_ms=ms, voxelize_ms=ms_vox)
