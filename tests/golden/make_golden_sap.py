"""Generates tests/golden/sap_golden.npz by RUNNING the reference's own DPSR and point_rasterize
(gaustudio/utils/graphics_utils.py) on the CPU.  The module is imported from the reference tree at generation time with
its marching-cubes import stubbed (neither cumcubes nor skimage is installed; the meshing is not recorded); nothing of
the reference is written into the repo, only inputs and outputs.

For a seeded sphere, a seeded torus and a plane patch (tests/sap_ref64.SHAPES) at res 32 and 64 it stores the
normals, the normalised points p (ShapeAsPoints' float32 transform of the shape's points, without the logit / sigmoid
round trip), the unweighted splat `raster_<res>` and DPSR's output `phi_<res>` (shifted and scaled, before the tanh
of generate_mesh), with sig = 2.  To keep the file small, the grids are kept on subgrids that span the whole grid:
`raster_32` whole [3,32,32,32], `raster_64` on every 2nd node [3,32,32,32], and phi on a [16,16,16] subgrid, every 2nd
node at res 32 and every 4th at res 64.

    python tests/golden/make_golden_sap.py        (needs /root/reference; CPU only)
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]
import sap_ref64  # noqa: E402

REF = "/root/reference/gaustudio/utils/graphics_utils.py"
OUT = os.path.join(HERE, "sap_golden.npz")


def reference_module():
    stub = types.ModuleType("skimage.measure")
    stub.marching_cubes = None
    sys.modules.setdefault("skimage", types.ModuleType("skimage")).measure = stub
    sys.modules["skimage.measure"] = stub
    spec = importlib.util.spec_from_file_location("ref_graphics_utils", REF)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    gu = reference_module()
    out = {}
    for name, make in sap_ref64.SHAPES.items():
        xyz, nrm = make()
        pts = torch.from_numpy(xyz)
        centre = pts.mean(dim=0)
        scale = (pts - centre).abs().max() * 1.2
        p = ((pts - centre) / scale + 1.0) / 2.0  # ShapeAsPoints.transform
        n = torch.from_numpy(nrm)
        out[f"{name}_normals"], out[f"{name}_p"] = nrm, p.numpy()
        for res in (32, 64):
            raster = gu.point_rasterize(p[None], n[None], (res,) * 3, weighted=False)[0].numpy()
            out[f"{name}_raster_{res}"] = raster if res == 32 else raster[:, ::2, ::2, ::2]
            dpsr = gu.DPSR(res=(res,) * 3, sig=2, scale=True, shift=True, weighted=False)
            with torch.no_grad():
                phi = dpsr(p[None], n[None])[0].numpy()
            k = res // 16
            out[f"{name}_phi_{res}"] = phi[::k, ::k, ::k]
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, sorted(out))


if __name__ == "__main__":
    main()
