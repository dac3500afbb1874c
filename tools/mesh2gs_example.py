"""Example: the gs-mesh2gs flow (gaustudio/scripts/mesh2gs.py:36-84) on this stack:
    python tools/mesh2gs_example.py --mesh mesh.ply --output_path gaussians.ply
Reads a binary little-endian mesh PLY (io.load_mesh_ply; textured meshes are not supported), paints it uniform 0.5
grey when it has no vertex colours, places 3 Gaussians per face with the `mesh` initializer into an SH-degree-1
model, and writes the 3DGS PLY.  Not part of the test suite (needs a GPU); every piece it calls is."""
import argparse, os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gaustudio_b200 import initializers, io
from gaustudio_b200.synthetic import GaussianPointCloud

ap = argparse.ArgumentParser()
ap.add_argument("--mesh", "-m", required=True); ap.add_argument("--output_path", "-o", required=True)
a = ap.parse_args()
dev = torch.device("cuda")
vertices, faces, colors = io.load_mesh_ply(a.mesh, device=dev)
if colors is None:
    print("No texture or face colors found. Using a uniform color.")
    colors = torch.full_like(vertices, 0.5)
gaussians = GaussianPointCloud.empty(sh_degree=1, device=dev)
initializers.make({"name": "mesh", "n_gaussians_per_surface_triangle": 3})(gaussians, (vertices, faces, colors))
io.export_ply(gaussians, a.output_path)
print(f"Gaussians exported to {a.output_path}")
