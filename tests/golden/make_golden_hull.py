"""Generates tests/golden/hull_golden.npz by RUNNING the reference's own code on the CPU: `Camera.insideView`,
`resizeTorch` / `resizeDepthTorch` through `Camera.downsample*` (gaustudio/datasets/__init__.py) and the float16 chain
of `DepthInitializer` (gaustudio/pipelines/initializers/depth.py: cache_dataset, process_dataset, build_model).  The
packages are imported from the reference tree at generation time; modules absent from this image are stubbed, and
trimesh by a recorder that keeps what would have been written.  Nothing of the reference is written into the repo,
only inputs and outputs.

    python tests/golden/make_golden_hull.py        (needs /root/reference; CPU only)

Contents:
  inside_*     three cameras (masks of two sizes, a 90-degree camera at the origin whose ndc = +-1 is exact in
               float32), points in and out of view, behind the cameras and on ndc = +-1; `inside_ref` [C,N] is
               insideView(points, mask) and `inside_nomask` [C,N] insideView(points)
  rs_*         an image, a mask and a depth map, downsample_scale(4) and downsample((20, 11)) of each
  dc_*         two views' world points, images, depth (zeros included) and fx, fy; the workspace's uint8 colours and
               float16 scales, and the model's xyz, rgb, log-scales and opacity as build_model hands them over
               (its `.cuda()` is the identity here, so rgb is the host's colour / 255)
"""
import importlib
import importlib.util
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "hull_golden.npz")
sys.path.insert(0, "/root/reference")


class _Stub(types.ModuleType):
    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return _Stub(self.__name__ + "." + name)

    def __call__(self, *a, **k):
        return _Stub("call")


def _import_with_stubs(name):
    for _ in range(80):
        try:
            return importlib.import_module(name)
        except ModuleNotFoundError as e:
            sys.modules[e.name] = _Stub(e.name)
    raise RuntimeError("too many missing modules")


class _Trimesh(types.ModuleType):
    """trimesh.PointCloud / load as depth.py uses them: export records the arrays, load returns them."""
    saved = {}

    class PointCloud:
        def __init__(self, vertices, colors=None):
            self.vertices = np.asarray(vertices, np.float64)  # trimesh keeps vertices as float64
            rgba = np.full((len(self.vertices), 4), 255, np.uint8)
            rgba[:, :3] = colors
            self.visual = types.SimpleNamespace(vertex_colors=rgba)

        def export(self, path):
            _Trimesh.saved[os.path.basename(path)] = self

    @staticmethod
    def load(path):
        return _Trimesh.saved[os.path.basename(path)]


def camera_look(Camera, pos, target, W, H, fovx, fovy):
    c = np.asarray(pos, np.float64)
    f = np.asarray(target, np.float64) - c
    f /= np.linalg.norm(f)
    right = np.cross(f, [0.0, 0.0, 1.0])
    right /= np.linalg.norm(right)
    R = np.stack([right, np.cross(f, right), f], axis=1)
    return R, -R.T @ c, Camera(R=R, T=-R.T @ c, FoVx=fovx, FoVy=fovy, image_width=W, image_height=H)


def inside_fixture(Camera, out):
    g = np.random.RandomState(11)
    cams = [((3.0, 0.5, 1.0), (0.0, 0.0, 0.0), 40, 30, 0.9, 0.7), ((-1.0, 2.5, -0.8), (0.1, 0.0, 0.2), 23, 17, 1.1, 0.85)]
    Rs, Ts, sizes, fovs, masks, ref, nomask = [], [], [], [], [], [], []
    objs = []
    for pos, tgt, W, H, fx, fy in cams:
        R, T, cam = camera_look(Camera, pos, tgt, W, H, fx, fy)
        objs.append((R, T, cam, W, H, fx, fy))
    # a camera at the origin looking down +z with a 90-degree field: clip_x = x and clip_w = z in float32
    cam0 = Camera(R=np.eye(3), T=np.zeros(3), FoVx=np.pi / 2, FoVy=np.pi / 2, image_width=23, image_height=17)
    objs.append((np.eye(3), np.zeros(3), cam0, 23, 17, np.pi / 2, np.pi / 2))
    pts = [g.uniform(-1.5, 1.5, (3000, 3))]
    z = g.uniform(0.5, 2.0, 64)
    y = g.uniform(-0.4, 0.4, 64) * z
    pts += [np.stack([s * z, y, z], 1) for s in (-1, 1)] + [np.stack([y, s * z, z], 1) for s in (-1, 1)]
    pts += [np.stack([y, y, -z], 1), np.stack([z, y, np.zeros_like(z)], 1)]  # behind and in the plane of camera 3
    pts = np.concatenate(pts).astype(np.float32)
    for R, T, cam, W, H, fx, fy in objs:
        m = (g.uniform(size=(H, W)) < 0.6).astype(np.float32)
        m[g.uniform(size=(H, W)) < 0.1] = 0.37  # nonzero fractions count as inside
        mt = torch.from_numpy(m)
        x = torch.from_numpy(pts)
        ref.append(cam.insideView(x, mt).numpy())
        nomask.append(cam.insideView(x).numpy())
        Rs.append(R); Ts.append(T); sizes.append((W, H)); fovs.append((fx, fy)); masks.append(m)
    out.update(inside_R=np.stack(Rs), inside_T=np.stack(Ts), inside_size=np.array(sizes), inside_fov=np.array(fovs),
               inside_points=pts, inside_ref=np.stack(ref), inside_nomask=np.stack(nomask),
               inside_proj=np.stack([o[2].full_proj_transform.numpy() for o in objs]))
    for i, m in enumerate(masks):
        out[f"inside_mask{i}"] = m


def resize_fixture(Camera, out):
    g = np.random.RandomState(12)
    H, W = 37, 53
    image = torch.from_numpy(g.uniform(size=(H, W, 3)).astype(np.float32))
    mask = torch.from_numpy((g.uniform(size=(H, W)) < 0.5).astype(np.float32))
    depth = torch.from_numpy(g.uniform(0.5, 4.0, (H, W)).astype(np.float32))
    depth[g.uniform(size=(H, W)) < 0.1] = 0.0
    out.update(rs_image=image.numpy(), rs_mask=mask.numpy(), rs_depth=depth.numpy())
    for tag, call in (("s4", lambda c: c.downsample_scale(4)), ("r2011", lambda c: c.downsample((20, 11)))):
        cam = Camera(R=np.eye(3), T=np.zeros(3), FoVx=1.0, FoVy=0.8, image_width=W, image_height=H)
        cam.image, cam.mask, cam.depth = image.clone(), mask.clone(), depth.clone()
        call(cam)
        out.update({f"rs_{tag}_image": cam.image.numpy(), f"rs_{tag}_mask": cam.mask.numpy(),
                    f"rs_{tag}_depth": cam.depth.numpy(), f"rs_{tag}_size": np.array([cam.image_width,
                                                                                      cam.image_height])})


class _View:
    """What cache_dataset reads from a camera after downsample_scale(4).to('cuda'): the given arrays."""

    def __init__(self, xyz, image, depth, fx, fy):
        self.xyz, self.image, self.depth = xyz, image, depth
        self.fx, self.fy = torch.tensor(fx, dtype=torch.float32), torch.tensor(fy, dtype=torch.float32)

    def downsample_scale(self, s):
        return self

    def to(self, dev):
        return self

    def depth2point(self, coordinate="camera"):
        return self.xyz


class _Model:
    def create_from_attribute(self, xyz, rgb, opacity, scale):
        self.got = dict(xyz=xyz, rgb=rgb, opacity=opacity, scale=scale)


def depth_fixture(out):
    sys.modules["trimesh"] = _Trimesh("trimesh")
    # depth.py and base.py alone, under a registry stub (the package's __init__ imports every initializer)
    root = "/root/reference/gaustudio/pipelines/initializers"
    pkg = types.ModuleType("gaustudio.pipelines.initializers")
    pkg.__path__, pkg.register = [root], lambda name: (lambda cls: cls)
    pipelines = types.ModuleType("gaustudio.pipelines")
    pipelines.__path__, pipelines.initializers = [], pkg
    sys.modules.update({"gaustudio.pipelines": pipelines, "gaustudio.pipelines.initializers": pkg})
    for name in ("base", "depth"):
        spec = importlib.util.spec_from_file_location(f"gaustudio.pipelines.initializers.{name}",
                                                      os.path.join(root, f"{name}.py"))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[spec.name] = mod
        for _ in range(20):
            try:
                spec.loader.exec_module(mod)
                break
            except ModuleNotFoundError as e:
                sys.modules[e.name] = _Stub(e.name)
    dmod = mod
    g = np.random.RandomState(13)
    views = []
    for i, (h, w) in enumerate(((9, 12), (7, 5))):
        xyz = torch.from_numpy(g.uniform(-3, 3, (h, w, 3)).astype(np.float32))
        img = torch.from_numpy(g.uniform(size=(h, w, 3)).astype(np.float32))
        img[0, :3] = torch.tensor([0.0, 1.0, 0.5])
        depth = torch.from_numpy(g.uniform(0.01, 6.0, (h, w)).astype(np.float32))
        depth[g.uniform(size=(h, w)) < 0.15] = 0.0
        fx, fy = float(g.uniform(5, 30)), float(g.uniform(5, 30))
        views.append(_View(xyz, img, depth, fx, fy))
        out.update({f"dc_xyz{i}": xyz.numpy(), f"dc_image{i}": img.numpy(), f"dc_depth{i}": depth.numpy(),
                    f"dc_f{i}": np.array([fx, fy], np.float32)})
    cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        with tempfile.TemporaryDirectory() as ws:
            init = dmod.DepthInitializer({"workspace_dir": ws})
            init.cache_dataset(views)
            init.process_dataset()
            scales16 = np.fromfile(os.path.join(ws, "scales.bin"), dtype=np.float16)
            model = _Model()
            init.build_model(model)
    finally:
        torch.Tensor.cuda = cuda
    pc = _Trimesh.saved["fused.ply"]
    m = model.got
    out.update(dc_points16=pc.vertices.astype(np.float16), dc_colors=pc.visual.vertex_colors[:, :3].copy(),
               dc_scales16=scales16, dc_model_xyz=m["xyz"].numpy(), dc_model_rgb=m["rgb"].numpy(),
               dc_model_log_scale=m["scale"].numpy(), dc_model_opacity=np.asarray(m["opacity"], np.float32))


def main():
    ds = _import_with_stubs("gaustudio.datasets")
    out = {}
    inside_fixture(ds.Camera, out)
    resize_fixture(ds.Camera, out)
    depth_fixture(out)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
