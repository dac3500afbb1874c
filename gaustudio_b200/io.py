"""On-disk formats either side of the path (SURVEY.md §8f rank 4) without `plyfile` / `omegaconf`:

* the 3DGS PLY point cloud as `BasePointCloud.load` reads it (`gaustudio/models/base.py:73-105`: one `vertex`
  element, float properties; attributes found by name prefix and ordered by their numeric suffix) and as
  `VanillaPointCloud.export` writes it (`gaustudio/models/vanilla_sg.py:144-181`: x y z nx ny nz f_dc_* f_rest_*
  opacity scale_* rot_*, little-endian float32, SH stored channel-major);
* `cameras.json` entries -> `Camera` (`gaustudio/utils/cameras_utils.py:8-38`).
"""
import json
import math
import re

import numpy as np
import torch

from .camera import Camera
from .synthetic import GaussianPointCloud

_PLY_TYPES = {"char": "i1", "uchar": "u1", "short": "i2", "ushort": "u2", "int": "i4", "uint": "u4", "float": "f4",
              "double": "f8", "int8": "i1", "uint8": "u1", "int16": "i2", "uint16": "u2", "int32": "i4", "uint32": "u4",
              "float32": "f4", "float64": "f8"}


def read_ply_vertices(path):
    """-> structured numpy array of the `vertex` element (ascii, binary_little_endian or binary_big_endian)."""
    with open(path, "rb") as f:
        if f.readline().strip() != b"ply":
            raise ValueError(f"{path}: not a PLY file")
        fmt, count, props, in_vertex = None, 0, [], False
        while True:
            line = f.readline()
            if not line:
                raise ValueError(f"{path}: unterminated PLY header")
            tok = line.decode("ascii", "replace").split()
            if not tok or tok[0] == "comment":
                continue
            if tok[0] == "format":
                fmt = tok[1]
            elif tok[0] == "element":
                if props and not in_vertex:
                    pass
                in_vertex = tok[1] == "vertex"
                if in_vertex:
                    count = int(tok[2])
                elif count:  # an element after `vertex`: stop collecting properties
                    in_vertex = False
            elif tok[0] == "property" and in_vertex:
                if tok[1] == "list":
                    raise ValueError("list properties are not supported in the vertex element")
                props.append((tok[2], _PLY_TYPES[tok[1]]))
            elif tok[0] == "end_header":
                break
        if fmt == "ascii":
            data = np.loadtxt(f, max_rows=count, ndmin=2)
            out = np.empty(count, dtype=[(n, t) for n, t in props])
            for i, (n, _) in enumerate(props):
                out[n] = data[:, i]
            return out
        order = "<" if fmt == "binary_little_endian" else ">"
        dt = np.dtype([(n, order + t) for n, t in props])
        return np.frombuffer(f.read(count * dt.itemsize), dtype=dt, count=count)


def _group(v, prefix):
    names = [n for n in v.dtype.names if n.startswith(prefix) and re.fullmatch(r".*_\d+", n)]
    names.sort(key=lambda n: int(n.split("_")[-1]))
    return np.stack([v[n] for n in names], axis=1).astype(np.float32) if names else None


def load_ply(path, sh_degree=3, active_sh_degree=0, device="cpu"):
    """PLY -> GaussianPointCloud holding the RAW attributes (log-scale, opacity logit, un-normalised rotation),
    `_f_dc` [P,3] and `_f_rest` [P,45] exactly as `BasePointCloud.load` stores them; `active_sh_degree` starts at
    0 like the reference model (`vanilla_sg.py:40`).  A vertex element with a `filter_3D` property (a Mip-Splatting
    checkpoint) gives a `MipPointCloud` carrying it as `filter_3D` [P,1]."""
    v = read_ply_vertices(path)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(device)
    xyz = np.stack([v["x"], v["y"], v["z"]], axis=1)
    f_dc, f_rest = _group(v, "f_dc"), _group(v, "f_rest")
    if f_rest is None:
        f_rest = np.zeros((len(v), 3 * ((sh_degree + 1) ** 2 - 1)), np.float32)
    args = (t(xyz), t(_group(v, "scale")), t(_group(v, "rot")), t(v["opacity"][:, None]), t(f_dc), t(f_rest))
    if "filter_3D" in v.dtype.names:
        from .mip import MipPointCloud
        return MipPointCloud(*args, sh_degree=sh_degree, active_sh_degree=active_sh_degree,
                             filter_3D=t(v["filter_3D"][:, None]))
    return GaussianPointCloud(*args, sh_degree=sh_degree, active_sh_degree=active_sh_degree)


def export_ply(model, path):
    """GaussianPointCloud -> PLY in the reference's export layout (binary little-endian float32); a model with a
    `filter_3D` (MipPointCloud) also writes it, last, as Mip-Splatting does."""
    n = len(model._xyz)
    flat = lambda a: a.detach().reshape(n, -1, 3).transpose(1, 2).flatten(start_dim=1).cpu().numpy()
    cols = [model._xyz.detach().cpu().numpy(), np.zeros((n, 3), np.float32), flat(model._f_dc), flat(model._f_rest),
            model._opacity.detach().reshape(n, 1).cpu().numpy(), model._scale.detach().cpu().numpy(),
            model._rot.detach().cpu().numpy()]
    names = ["x", "y", "z", "nx", "ny", "nz"]
    names += [f"f_dc_{i}" for i in range(cols[2].shape[1])] + [f"f_rest_{i}" for i in range(cols[3].shape[1])]
    names += ["opacity"] + [f"scale_{i}" for i in range(cols[5].shape[1])] + [f"rot_{i}" for i in range(cols[6].shape[1])]
    if getattr(model, "filter_3D", None) is not None:
        cols.append(model.filter_3D.detach().reshape(n, 1).cpu().numpy())
        names.append("filter_3D")
    data = np.concatenate(cols, axis=1).astype("<f4")
    header = "ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % n
    header += "".join(f"property float {nm}\n" for nm in names) + "end_header\n"
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        f.write(data.tobytes())


_SCAFFOLD_MLPS = (("mlp_opacity", "opacity_mlp.pt"), ("mlp_cov", "cov_mlp.pt"), ("mlp_color", "color_mlp.pt"),
                  ("mlp_feature_bank", "feature_bank_mlp.pt"))


def _plain_mlp(path, device):
    """A TorchScript MLP (Linear, ReLU, Linear[, activation]) as a plain nn.Sequential with its `0.*` / `2.*` weights;
    the activation is the module the traced one ends with."""
    from torch import nn
    ts = torch.jit.load(path, map_location="cpu")
    sd = ts.state_dict()
    w0, w2 = sd["0.weight"], sd["2.weight"]
    layers = [nn.Linear(w0.shape[1], w0.shape[0]), nn.ReLU(True), nn.Linear(w2.shape[1], w2.shape[0])]
    tail = [getattr(ts, n).original_name for n, _ in ts.named_children()][3:]
    acts = {"Tanh": nn.Tanh(), "Sigmoid": nn.Sigmoid(), "Softmax": nn.Softmax(dim=1)}
    for name in tail:
        if name not in acts:
            raise ValueError(f"{path}: unsupported layer {name} after the second Linear")
        layers.append(acts[name])
    mlp = nn.Sequential(*layers)
    mlp.load_state_dict({k: v for k, v in sd.items() if k.split(".")[0] in ("0", "2")})
    return mlp.to(device)


def load_scaffold(ply_path, mlp_dir=None, device="cpu"):
    """A Scaffold-GS checkpoint -> ScaffoldPointCloud.  The PLY's vertex element holds x y z nx ny nz f_offset_*
    f_anchor_feat_* opacity scale_0..5 rot_0..3, the offsets channel-major (f_offset_{c*k+j} is channel c of offset j);
    `mlp_dir` (default: the PLY's directory) holds the TorchScript MLPs opacity_mlp.pt, cov_mlp.pt, color_mlp.pt and
    optionally feature_bank_mlp.pt, whose weights are copied into plain modules."""
    import os
    from .scaffold import ScaffoldPointCloud
    v = read_ply_vertices(ply_path)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(device)
    n = len(v)
    offset = _group(v, "f_offset")
    if offset is None or offset.shape[1] % 3:
        raise ValueError(f"{ply_path}: no f_offset_* columns, or not a multiple of 3")
    offset = offset.reshape(n, 3, -1).transpose(0, 2, 1)
    mlp_dir = os.path.dirname(os.path.abspath(ply_path)) if mlp_dir is None else mlp_dir
    mlps = {}
    for attr, fname in _SCAFFOLD_MLPS:
        p = os.path.join(mlp_dir, fname)
        if os.path.exists(p):
            mlps[attr] = _plain_mlp(p, device)
        elif attr != "mlp_feature_bank":
            raise FileNotFoundError(p)
    return ScaffoldPointCloud(t(np.stack([v["x"], v["y"], v["z"]], axis=1)), t(offset), t(_group(v, "f_anchor_feat")),
                              t(v["opacity"][:, None]), t(_group(v, "scale")), t(_group(v, "rot")), **mlps)


def export_scaffold(model, ply_path):
    """ScaffoldPointCloud -> the layout load_scaffold reads: the PLY (binary little-endian float32) and, next to it, the
    MLPs traced to TorchScript on the CPU."""
    import copy
    import os
    n = model.num_points
    cols = [model._anchor, torch.zeros(n, 3), model._offset.transpose(1, 2).reshape(n, -1), model._anchor_feat,
            model._opacity.reshape(n, 1), model._scale, model._rot]
    cols = [c.detach().cpu().numpy().astype("<f4") for c in cols]
    names = ["x", "y", "z", "nx", "ny", "nz"] + [f"f_offset_{i}" for i in range(cols[2].shape[1])]
    names += [f"f_anchor_feat_{i}" for i in range(cols[3].shape[1])] + ["opacity"]
    names += [f"scale_{i}" for i in range(6)] + [f"rot_{i}" for i in range(4)]
    header = "ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % n
    header += "".join(f"property float {nm}\n" for nm in names) + "end_header\n"
    with open(ply_path, "wb") as f:
        f.write(header.encode("ascii"))
        f.write(np.concatenate(cols, axis=1).astype("<f4").tobytes())
    out_dir = os.path.dirname(os.path.abspath(ply_path))
    for attr, fname in _SCAFFOLD_MLPS:
        mlp = getattr(model, attr)
        if mlp is None:
            continue
        m = copy.deepcopy(mlp).cpu().eval()
        x = torch.rand(1, m[0].in_features)
        torch.jit.trace(m, x).save(os.path.join(out_dir, fname))


def export_points_ply(path, xyz, rgb=None, normals=None):
    """Surface point cloud (the `fused.ply` of gaustudio/scripts/extract_pcd.py:339-352, written there through
    open3d's `write_point_cloud`): binary little-endian, double x y z [nx ny nz] + uchar red green blue, the property
    layout open3d emits.  Tensors or arrays; colours in [0, 1], or uint8 colours written as they are."""
    def host(a):
        return None if a is None else np.asarray(a.detach().cpu() if isinstance(a, torch.Tensor) else a)
    xyz, rgb, normals = host(xyz), host(rgb), host(normals)
    n = xyz.shape[0]
    fields = [("x", "<f8"), ("y", "<f8"), ("z", "<f8")]
    if normals is not None:
        fields += [("nx", "<f8"), ("ny", "<f8"), ("nz", "<f8")]
    if rgb is not None:
        fields += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
    rec = np.empty(n, dtype=fields)
    for i, k in enumerate("xyz"):
        rec[k] = xyz[:, i]
    if normals is not None:
        for i, k in enumerate(("nx", "ny", "nz")):
            rec[k] = normals[:, i]
    if rgb is not None:
        c = rgb if rgb.dtype == np.uint8 else \
            np.clip(np.nan_to_num(rgb.astype(np.float64)) * 255.0, 0, 255).astype(np.uint8)  # open3d truncates
        for i, k in enumerate(("red", "green", "blue")):
            rec[k] = c[:, i]
    names = {"<f8": "double", "u1": "uchar"}
    head = ["ply", "format binary_little_endian 1.0", f"element vertex {n}"] + \
           [f"property {names[t]} {k}" for k, t in fields] + ["end_header"]
    with open(path, "wb") as f:
        f.write(("\n".join(head) + "\n").encode("ascii"))
        f.write(rec.tobytes())


def export_mesh_ply(path, vertices, faces, colors=None):
    """Triangle mesh (the `fused_mesh.ply` of gaustudio/scripts/extract_mesh.py:146, written there through trimesh):
    binary little-endian, double x y z per vertex and `property list uchar int vertex_indices` per face.  With
    `colors` ([V,3] in [0, 1], the textured mesh of texture_mesh.py:143-145) each vertex also gets uchar red green blue
    alpha, rint(255 c) and alpha 255, as trimesh writes vertex colours.  Tensors or arrays."""
    host = lambda a: np.asarray(a.detach().cpu() if isinstance(a, torch.Tensor) else a)
    v, f = host(vertices).reshape(-1, 3), host(faces).reshape(-1, 3)
    rec = np.empty(len(f), dtype=[("n", "u1"), ("i", "<i4", (3,))])
    rec["n"] = 3
    rec["i"] = f
    vprops = ["property double x", "property double y", "property double z"]
    if colors is None:
        vdata = v.astype("<f8")
    else:
        c = host(colors).reshape(-1, 3).astype(np.float64)
        vdata = np.empty(len(v), dtype=[("xyz", "<f8", (3,)), ("rgba", "u1", (4,))])
        vdata["xyz"] = v
        vdata["rgba"][:, :3] = np.clip(np.rint(np.nan_to_num(c) * 255.0), 0, 255).astype(np.uint8)
        vdata["rgba"][:, 3] = 255
        vprops += [f"property uchar {k}" for k in ("red", "green", "blue", "alpha")]
    head = ["ply", "format binary_little_endian 1.0", f"element vertex {len(v)}", *vprops, f"element face {len(f)}",
            "property list uchar int vertex_indices", "end_header"]
    with open(path, "wb") as fh:
        fh.write(("\n".join(head) + "\n").encode("ascii"))
        fh.write(vdata.tobytes())
        fh.write(rec.tobytes())


def load_mesh_ply(path, device="cpu"):
    """Binary little-endian triangle mesh PLY, as export_mesh_ply, trimesh and open3d write it: a `vertex` element with
    float or double x y z (other scalar properties skipped; uchar red green blue read as colours) and a `face` element
    whose only property is a list of uchar count and int / uint indices, every count 3.
    -> (vertices [V,3] float32, faces [F,3] int64, colors [V,3] float32 in [0, 1] or None), tensors on `device`."""
    with open(path, "rb") as fh:
        if fh.readline().strip() != b"ply":
            raise ValueError(f"{path}: not a PLY file")
        elements, fmt = [], None
        while True:
            line = fh.readline()
            if not line:
                raise ValueError(f"{path}: unterminated PLY header")
            tok = line.decode("ascii", "replace").split()
            if not tok or tok[0] in ("comment", "obj_info"):
                continue
            if tok[0] == "format":
                fmt = tok[1]
            elif tok[0] == "element":
                elements.append((tok[1], int(tok[2]), []))
            elif tok[0] == "property":
                elements[-1][2].append(tok[1:])
            elif tok[0] == "end_header":
                break
        if fmt != "binary_little_endian":
            raise ValueError(f"{path}: only binary_little_endian meshes are supported, not {fmt}")
        verts = faces = colors = None
        for name, count, props in elements:
            if name == "vertex":
                if any(p[0] == "list" for p in props):
                    raise ValueError(f"{path}: list properties are not supported in the vertex element")
                dt = np.dtype([(p[1], "<" + _PLY_TYPES[p[0]]) for p in props])
                rec = np.frombuffer(fh.read(count * dt.itemsize), dtype=dt, count=count)
                verts = np.stack([rec[k] for k in "xyz"], axis=1).astype(np.float32)
                if all(k in dt.names for k in ("red", "green", "blue")):
                    colors = np.stack([rec[k] for k in ("red", "green", "blue")], axis=1).astype(np.float32) / 255.0
            elif name == "face":
                if len(props) != 1 or props[0][0] != "list" or props[0][1] not in ("uchar", "uint8") or \
                        props[0][2] not in ("int", "uint", "int32", "uint32"):
                    raise ValueError(f"{path}: the face element must be one list of uchar count and int indices")
                dt = np.dtype([("n", "u1"), ("i", "<" + _PLY_TYPES[props[0][2]], (3,))])
                rec = np.frombuffer(fh.read(count * dt.itemsize), dtype=dt, count=count)
                if (rec["n"] != 3).any():
                    raise ValueError(f"{path}: only triangle faces are supported")
                faces = rec["i"].astype(np.int64)
            else:
                raise ValueError(f"{path}: unsupported PLY element {name!r}")
    if verts is None or faces is None:
        raise ValueError(f"{path}: a mesh PLY needs a vertex and a face element")
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(device)
    return t(verts), t(faces.reshape(-1, 3)), t(colors)


def camera_from_json(entry):
    """One `cameras.json` entry (id, img_name, width, height, position, rotation (camera-to-world), fx, fy)."""
    c2w = np.eye(4)
    c2w[:3, :3] = np.array(entry["rotation"])
    c2w[:3, 3] = np.array(entry["position"])
    w2c = np.linalg.inv(c2w)
    fov = lambda focal, pixels: 2 * math.atan(pixels / (2 * focal))
    return Camera(R=w2c[:3, :3].transpose(), T=w2c[:3, 3], FoVx=fov(entry["fx"], entry["width"]),
                  FoVy=fov(entry["fy"], entry["height"]), image_width=entry["width"], image_height=entry["height"])


def load_cameras_json(path):
    with open(path) as f:
        return [camera_from_json(e) for e in json.load(f)]
