"""Example: the gs-extract-pcd flow of the reference (gaustudio/scripts/extract_pcd.py) on this stack:
    python tools/extract_pcd_example.py --model point_cloud.ply --camera cameras.json [--sh 0] [-o fused.ply]
                                        [--meshing {sap,none}] [--clean]
Loads a 3DGS PLY and cameras.json (gaustudio_b200.io), renders every view with the vanilla renderer, runs the GPU
post-pass (masked bilateral filter, normals, fusion) and writes the oriented surface point cloud.  With `--meshing sap`
(the default, as in the reference) it then meshes that cloud with Shape-as-Points (extract.mesh_sap, res 256, sig 2) and
writes fused_mesh.ply beside it.  The reference always cleans the fused cloud first (clean_point_cloud: statistical,
then normal outlier removal); here that step is opt-in with `--clean` (extract.clean_point_cloud on the unfiltered cloud,
NaN normals included, before fused.ply is written and meshed, as at extract_pcd.py:369-399).  Without it, the rows with
a NaN normal are dropped instead, and nothing else is removed.  With no model it runs on
a synthetic scene.  Not part of the test suite (needs a GPU); every piece it calls is."""
import argparse, os, sys
import torch
sys.path.insert(0, ".")
from gaustudio_b200 import extract, io, renderers
from gaustudio_b200.synthetic import build_config

ap = argparse.ArgumentParser()
ap.add_argument("--model", "-m"); ap.add_argument("--camera", "-c"); ap.add_argument("--sh", type=int, default=0)
ap.add_argument("--output", "-o", default="fused.ply")
ap.add_argument("--meshing", choices=["sap", "none"], default="sap")
ap.add_argument("--clean", action="store_true", help="statistical + normal outlier removal, as the reference does")
a = ap.parse_args()
dev = torch.device("cuda")
if a.model:
    pcd = io.load_ply(a.model, active_sh_degree=a.sh, device=dev)
    cameras = io.load_cameras_json(a.camera)
else:
    pcd, cameras, _ = build_config("cfg1", P=50000, W=320, H=240, K=12)
    pcd.to(dev); pcd.active_sh_degree = a.sh
cameras = [c.to(dev) for c in cameras]
renderer = renderers.make({"name": "vanilla_renderer"})
xyz, rgb, normals, _ = extract.extract_pcd(renderer, pcd, cameras)
if a.clean:
    n_fused = xyz.shape[0]
    xyz, rgb, normals, _ = extract.clean_point_cloud(xyz.detach().float().contiguous(), rgb,
                                                     normals.float().contiguous())
    print(f"cleaning kept {xyz.shape[0]} of {n_fused} fused points")
else:
    keep = ~torch.isnan(normals).any(1)
    xyz, rgb, normals = xyz[keep], rgb[keep], normals[keep]
io.export_points_ply(a.output, xyz, rgb, normals)
print(f"{xyz.shape[0]} surface points from {len(cameras)} views -> {a.output}")
if a.meshing == "sap":
    vertices, faces = extract.mesh_sap(xyz.detach().contiguous(), normals.contiguous())
    mesh_path = os.path.join(os.path.dirname(os.path.abspath(a.output)), "fused_mesh.ply")
    io.export_mesh_ply(mesh_path, vertices, faces)
    print(f"{vertices.shape[0]} vertices, {faces.shape[0]} faces -> {mesh_path}")
