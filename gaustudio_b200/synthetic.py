"""Seeded synthetic scenes + cameras for BASELINE.json's configs (SURVEY.md §8d).

The Gaussian container mirrors the consumer contract of the reference model
`gaustudio/models/vanilla_sg.py:19-141` (`VanillaPointCloud`): raw attributes
`_xyz,_scale,_rot,_opacity,_f_dc,_f_rest`, `get_attribute(name)` applying the
activations exp / sigmoid / normalize (`vanilla_sg.py:58-63`, `models/utils.py:6-32`),
`get_features` = cat(f_dc, f_rest) as [P,16,3] (`vanilla_sg.py:102-106`),
`active_sh_degree`, `max_sh_degree`.  No PLY I/O (out of scope, SURVEY.md §8f rank 4).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from .camera import Camera, orbit_cameras


class GaussianPointCloud(torch.nn.Module):
    activations = {"scale": torch.exp, "opacity": torch.sigmoid, "rot": lambda r: F.normalize(r)}

    def __init__(self, xyz, scale, rot, opacity, f_dc, f_rest, sh_degree=3, active_sh_degree=None):
        super().__init__()
        self._xyz, self._scale, self._rot, self._opacity = xyz, scale, rot, opacity
        self._f_dc, self._f_rest = f_dc, f_rest
        self.max_sh_degree = sh_degree
        self.active_sh_degree = sh_degree if active_sh_degree is None else active_sh_degree
        self.num_points = xyz.shape[0]

    def get_attribute(self, name):
        v = getattr(self, "_" + name)
        return self.activations[name](v) if name in self.activations else v

    @property
    def get_features(self):
        n = len(self._f_dc)
        dc, rest = math.prod(self._f_dc.shape[1:]) // 3, math.prod(self._f_rest.shape[1:]) // 3  # also at P = 0
        return torch.cat((self._f_dc.reshape(n, dc, 3), self._f_rest.reshape(n, rest, 3)), dim=1)

    _ATTRS = ("_xyz", "_scale", "_rot", "_opacity", "_f_dc", "_f_rest")

    def to(self, device):
        for k in self._ATTRS:
            v = getattr(self, k)
            if isinstance(v, torch.nn.Parameter):  # registered by an optimizer plugin: move in place, stay a leaf
                v.data = v.data.to(device)
            else:
                setattr(self, k, v.to(device))
        return self

    def requires_grad_(self, flag=True):
        for k in self._ATTRS:
            v = getattr(self, k)
            if isinstance(v, torch.nn.Parameter):
                v.requires_grad_(flag)
            else:
                setattr(self, k, v.detach().requires_grad_(flag))
        return self

    def parameters_list(self):
        return [self._xyz, self._scale, self._rot, self._opacity, self._f_dc, self._f_rest]

    @classmethod
    def empty(cls, sh_degree=3, device="cuda"):
        """A model with no Gaussians and active_sh_degree 0, as VanillaPointCloud.__init__ leaves it
        (vanilla_sg.py:39-40); fill it with create_from_attribute or an initializer."""
        z = lambda *shape: torch.zeros(*shape, dtype=torch.float32, device=device)
        return cls(z(0, 3), z(0, 3), z(0, 4), z(0, 1), z(0, 1, 3), z(0, (sh_degree + 1) ** 2 - 1, 3), sh_degree, 0)

    def create_from_attribute(self, xyz, rgb=None, scale=None, rot=None, opacity=None):
        """vanilla_sg.py:69-97: replace the six attributes in place on the model's device.  Inputs are numpy arrays
        or tensors, converted to float32: xyz [P,3]; rgb [P,3] in [0, 1] (None: ones) -> _f_dc = RGB2SH(rgb)
        [P,1,3]; _f_rest zeros; scale [P,3] log-scales (None: log(sqrt(dist2(xyz) + 1e-7)) on all three axes, which
        needs a CUDA model); rot [P,4] (None: (1, 0, 0, 0)); opacity [P,1] logits (None: inverse_sigmoid(0.1))."""
        dev = self._xyz.device
        host = [_float_rows(xyz, "xyz", 3)]
        P = host[0].shape[0]
        for a, name, w in ((rgb, "rgb", 3), (scale, "scale", 3), (rot, "rot", 4), (opacity, "opacity", 1)):
            host.append(None if a is None else _float_rows(a, name, w, P))
        if scale is None and dev.type != "cuda" and P > 0:
            raise ValueError("scale=None needs dist2, which has no CPU path: move the model to a CUDA device")
        x, rgb, scale, rot, opacity = (None if a is None else a.to(dev) for a in host)
        if rgb is None:
            rgb = torch.ones_like(x)
        f_dc = ((rgb - 0.5) / SH_C0).unsqueeze(-1).transpose(1, 2).contiguous()
        if scale is None:
            from .initializers import dist2
            scale = torch.log(torch.sqrt(dist2(x) + 1e-7))[..., None].repeat(1, 3)
        if rot is None:
            rot = torch.zeros((P, 4), dtype=torch.float32, device=dev)
            rot[:, 0] = 1
        if opacity is None:
            o = 0.1 * torch.ones((P, 1), dtype=torch.float32, device=dev)
            opacity = torch.log(o / (1 - o))
        self._set_attributes(x, f_dc, scale, rot, opacity)
        return self

    def _set_attributes(self, xyz, f_dc, scale, rot, opacity):
        """Replaces the six attributes.  An attribute that is an nn.Parameter (a model already set up for training)
        becomes a new Parameter with the same requires_grad: the old one, and any optimizer state keyed on it, no
        longer belongs to the model, so build the optimizer after (re-)initialising."""
        P = xyz.shape[0]
        f_rest = torch.zeros((P, (self.max_sh_degree + 1) ** 2 - 1, 3), dtype=torch.float32, device=xyz.device)
        for k, v in zip(self._ATTRS, (xyz, scale, rot, opacity, f_dc, f_rest)):
            old = getattr(self, k, None)
            setattr(self, k, torch.nn.Parameter(v, requires_grad=old.requires_grad)
                    if isinstance(old, torch.nn.Parameter) else v)
        self.num_points = P


SH_C0 = 0.28209479177387814  # RGB2SH of gaustudio/utils/sh_utils.py


def _float_rows(a, name, width, rows=None):
    """numpy array or tensor [rows, width] of real numbers -> float32 tensor on its own device (host for numpy)."""
    if isinstance(a, np.ndarray):
        a = torch.from_numpy(np.ascontiguousarray(a))
    if not isinstance(a, torch.Tensor):
        raise ValueError(f"{name} must be a numpy array or a tensor")
    if a.dtype == torch.bool or a.is_complex() or not (a.is_floating_point() or a.dtype in
                                                         (torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64)):
        raise ValueError(f"{name} must hold real numbers, got {a.dtype}")
    if a.dim() != 2 or a.shape[1] != width or (rows is not None and a.shape[0] != rows):
        want = f"[{'P' if rows is None else rows},{width}]"
        raise ValueError(f"{name} must be {want}, got {tuple(a.shape)}")
    return a.detach().to(torch.float32)


def _ball(g, n, rho):
    d = torch.randn(n, 3, generator=g)
    d = d / d.norm(dim=1, keepdim=True)
    return d * (rho * torch.rand(n, 1, generator=g) ** (1.0 / 3.0))


def make_scene(P, rho, s0, seed, sh_degree=3):
    """Uniform ball of radius rho; log-scales N(log s0, 0.5^2); rot N(0,I); opacity logits N(0,2^2);
    f_dc N(0,1), f_rest N(0,0.1^2) (SURVEY.md §8d 'Synthetic scene generator')."""
    g = torch.Generator().manual_seed(seed)
    xyz = _ball(g, P, rho)
    scale = math.log(s0) + 0.5 * torch.randn(P, 3, generator=g)
    rot = torch.randn(P, 4, generator=g)
    opacity = 2.0 * torch.randn(P, 1, generator=g)
    nrest = (sh_degree + 1) ** 2 - 1
    f_dc = torch.randn(P, 1, 3, generator=g)
    f_rest = 0.1 * torch.randn(P, nrest, 3, generator=g)
    return GaussianPointCloud(xyz, scale, rot, opacity, f_dc, f_rest, sh_degree)


def make_unbounded_scene(P, seed, sh_degree=3):
    """cfg 5: 30 % in the unit ball (s0=0.008), 70 % in a shell r in [2,30] log-uniform, scale ∝ r."""
    g = torch.Generator().manual_seed(seed)
    n0 = int(0.3 * P)
    n1 = P - n0
    xyz0 = _ball(g, n0, 1.0)
    d = torch.randn(n1, 3, generator=g)
    d = d / d.norm(dim=1, keepdim=True)
    r = torch.exp(math.log(2.0) + (math.log(30.0) - math.log(2.0)) * torch.rand(n1, 1, generator=g))
    xyz = torch.cat([xyz0, d * r])
    base = torch.cat([torch.full((n0, 1), math.log(0.008)), torch.log(0.008 * r)])
    scale = base + 0.5 * torch.randn(P, 3, generator=g)
    rot = torch.randn(P, 4, generator=g)
    opacity = 2.0 * torch.randn(P, 1, generator=g)
    nrest = (sh_degree + 1) ** 2 - 1
    f_dc = torch.randn(P, 1, 3, generator=g)
    f_rest = 0.1 * torch.randn(P, nrest, 3, generator=g)
    return GaussianPointCloud(xyz, scale, rot, opacity, f_dc, f_rest, sh_degree)


def _fov(size, focal):
    return 2.0 * math.atan(size / (2.0 * focal))


# name -> dict(scene=..., cameras(K, indices) -> list[Camera]); numbers from SURVEY.md §8d / BASELINE.md §3
CONFIGS = {
    "cfg1": dict(P=10_000, rho=1.0, s0=0.03, seed=1, W=256, H=256, fovy=math.radians(49.1), fovx=math.radians(49.1),
                 radius=3.0, elev=30.0, K=1),
    "cfg2": dict(P=100_000, rho=1.3, s0=0.02, seed=2, W=800, H=800, fovy=0.6911, fovx=0.6911, radius=4.03, elev=30.0,
                 K=100),
    "cfg3": dict(P=1_000_000, rho=1.0, s0=0.005, seed=3, W=1920, H=1080, fovy=math.radians(49.1),
                 fovx=_fov(1920, 1080 / (2 * math.tan(math.radians(49.1) / 2))), radius=3.0, elev=30.0, K=200),
    "cfg4": dict(P=1_000_000, rho=1.0, s0=0.005, seed=3, W=1920, H=1080, fovy=math.radians(49.1),
                 fovx=_fov(1920, 1080 / (2 * math.tan(math.radians(49.1) / 2))), radius=3.0, elev=30.0, K=800),
    "cfg5": dict(P=5_000_000, seed=5, W=1440, H=1080, fovy=math.radians(49.1),
                 fovx=_fov(1440, 1080 / (2 * math.tan(math.radians(49.1) / 2))), radius=4.0, elev=15.0, K=200,
                 unbounded=True),
}


def build_config(name, P=None, K=None, W=None, H=None):
    """(model, cameras, cfg) for a named BASELINE config; P / K / resolution can be scaled down for tests
    (focal length scales with the resolution so the framing is preserved)."""
    c = dict(CONFIGS[name])
    if P is not None:
        c["P"] = P
    if K is not None:
        c["K"] = K
    if W is not None or H is not None:
        W = W or c["W"]
        H = H or c["H"]
        fy = c["H"] / (2 * math.tan(c["fovy"] / 2)) * (H / c["H"])
        c.update(W=W, H=H, fovy=_fov(H, fy), fovx=_fov(W, fy))
    if c.get("unbounded"):
        model = make_unbounded_scene(c["P"], c["seed"])
    else:
        model = make_scene(c["P"], c["rho"], c["s0"], c["seed"])
    cams = orbit_cameras(c["K"], c["radius"], c["elev"], c["W"], c["H"], c["fovx"], c["fovy"])
    return model, cams, c
