"""A/B of the compositing-kernel variants selected by environment variables read once per process (GSR_BWD_NSUB = pixels
per lane of the backward: 1 or 2; GSR_FWD_TMA=1 = TMA bulk-copy staging in the forward), one subprocess per variant.
(Up to commit a9bd034 the backward also had 4 / 8 pixels per lane and a second occupancy target per variant --
`GSR_BWD_MINB`; those measurements are in profiles/r2_ab_bwd_variants.json.)  For each variant: forward
outputs must be BIT-IDENTICAL to the unmodified reference extension (oracle/_ref) and the gradients within 1e-3
relative of the reference's, then per-kernel CUDA-event times over a few views.
Usage: python tools/render_ab.py [cfg3] ["1 2"]"""
import json, os, subprocess, sys, tempfile

CHILD = r'''
import sys, ctypes, json, math, torch
sys.path.insert(0, "."); sys.path.insert(0, "tests")
from gaustudio_b200 import renderers, _lib
from gaustudio_b200.rasterizer import GaussianRasterizationSettings, GaussianRasterizer
from gaustudio_b200.synthetic import build_config
from oracle import ref_driver
name, out = sys.argv[1], sys.argv[2]
model, cams, c = build_config(name, K=8); dev = torch.device("cuda"); model.to(dev).requires_grad_(True)
L = _lib.lib()
res = {}
# ---- parity of one view against the compiled reference (un-fused on both sides: identical inputs)
cam = cams[0].to(dev)
def run(rast):
    for p in model.parameters_list(): p.grad = None
    rs = GaussianRasterizationSettings(c["H"], c["W"], math.tan(cam.FoVx * .5), math.tan(cam.FoVy * .5), torch.zeros(3, device=dev),
                                       1.0, cam.world_view_transform, cam.full_proj_transform, 3, cam.camera_center, False, False)
    m2d = torch.zeros_like(model._xyz, requires_grad=True)
    o = rast(rs, model.get_attribute("xyz"), m2d, model.get_attribute("opacity"), shs=model.get_features,
             scales=model.get_attribute("scale"), rotations=model.get_attribute("rot"))
    color, radii, depth, median, opac = o
    g = torch.Generator().manual_seed(7)
    loss = sum((t * torch.randn(t.shape, generator=g).to(dev)).sum() for t in (color, depth, median, opac))
    loss.backward()
    return [t.detach().clone() for t in (color, radii, depth, median, opac)], [m2d.grad.clone()] + [p.grad.clone() for p in model.parameters_list()]
fo, go = run(lambda rs, *a, **k: GaussianRasterizer(rs)(*a, **k))
if ref_driver.available():
    fr, gr = run(ref_driver.rasterize)
    res["fwd_bit_identical"] = all(torch.equal(a, b) for a, b in zip(fo, fr))
    worst = 0.0
    for a, b in zip(go, gr):
        scale = b.abs().max().clamp_min(1e-30)
        worst = max(worst, float(((a - b).abs() - 1e-3 * b.abs()).clamp_min(0).max() / scale))
    res["grad_excess_over_1e-3rel_in_units_of_scale"] = worst
# ---- times (fused path, like the bench)
r = renderers.make({"name": "vanilla_renderer", "fused_activations": True})
for i in range(8):
    if i == 3: torch.cuda.synchronize(); L.gsr_profile_enable(1)
    o = r.render(cams[i].to(dev), model)
    loss = o["render"].abs().mean() + 0.1 * o["rendered_depth"].abs().mean() + 0.1 * o["rendered_final_opacity"].abs().mean()
    loss.backward()
torch.cuda.synchronize()
ms = (ctypes.c_float * 8)(); cn = (ctypes.c_int * 8)(); L.gsr_profile_read(ms, cn)
names = ["preprocess_fwd", "tile_scan", "scatter", "tile_sort", "render_fwd", "render_bwd", "preprocess_bwd", "depth2normal"]
res["ms"] = {n: round(ms[i] / max(cn[i], 1), 4) for i, n in enumerate(names) if cn[i]}
json.dump(res, open(out, "w"))
'''

name = sys.argv[1] if len(sys.argv) > 1 else "cfg3"
variants = (sys.argv[2] if len(sys.argv) > 2 else "1 2").split()
rep = {"config": name, "variants": {}}
with tempfile.TemporaryDirectory() as d:
    for v in variants:
        nsub, _, minb = v.partition(":")
        env = dict(os.environ, GSR_BWD_NSUB=nsub, GSR_BWD_MINB=minb or "0")
        path = os.path.join(d, "r.json")
        try:
            subprocess.run([sys.executable, "-c", CHILD, name, path], check=True, env=env, timeout=900)
            rep["variants"][v] = json.load(open(path))
        except Exception as ex:  # noqa: BLE001
            rep["variants"][v] = {"error": str(ex)}
print(json.dumps(rep))
