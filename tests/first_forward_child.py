"""Child process of tests/test_gpu_first_forward.py: ONE first forward of a fresh process, its state, two re-renders.

    python tests/first_forward_child.py --case <name> --scene <cfg5|cfg1|B> --out <file.npz>

The scene is built on the CPU before any CUDA work.  The rasterizer inputs are then produced on the device the way the
case prescribes and the forward is issued AT ONCE (no synchronisation between producing and rendering).  A recording
shim around `_C.rasterize_gaussians` / `_C.rasterize_surfels` keeps the exact arguments the forward was given and what
it returned (it adds no CUDA work).  Right after the forward its internal state is exported (`_C.debug_export`); only
then does the process synchronise, download the inputs, and render twice more from the same device tensors: render 2
takes the speculative form (a hint exists now), render 3 the plain blocking form the first one took
(`set_speculation(False)`).  Everything goes into the npz; nothing is asserted here -- the parent judges."""
import argparse
import contextlib
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

CASES = ("materialised", "same_stream", "same_stream_fused", "side_stream_waited", "non_default_stream",
         "after_allocator_churn", "eager_modules", "mip", "surfel")
# positional arguments of _C.rasterize_gaussians that are tensors, by name
ARG_NAMES = ("bg", "means3D", "colors_precomp", "opacities", "scales", "rotations", "scale_modifier", "cov3D_precomp",
             "viewmatrix", "projmatrix", "tanfovx", "tanfovy", "H", "W", "shs", "D", "campos", "prefiltered", "debug")
# _C.rasterize_surfels has no cov3D_precomp
SURFEL_ARG_NAMES = tuple(n for n in ARG_NAMES if n != "cov3D_precomp")
EXPORT_KEYS = ("means2D", "conic_opacity", "depths", "rgb", "cov3D", "clamped", "tiles_touched", "ranges", "point_list",
               "n_contrib", "final_T")


class Recorder:
    """Stands in for a function of gaustudio_b200._C and keeps (args, kwargs, result) of every call."""

    def __init__(self, module, name):
        self.orig, self.calls = getattr(module, name), []
        setattr(module, name, self)

    def __call__(self, *a, **kw):
        out = self.orig(*a, **kw)
        self.calls.append((a, kw, out))
        return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--case", required=True, choices=CASES)
    ap.add_argument("--scene", default="cfg5", choices=("cfg5", "cfg1", "B"))
    ap.add_argument("--out", required=True)
    a = ap.parse_args()

    import numpy as np
    import torch

    from gaustudio_b200 import _C, _lib, renderers
    from gaustudio_b200.synthetic import GaussianPointCloud, build_config

    case, out, rounded = a.case, {}, []  # rounded: the inputs that an activation on the device produces
    kind = case if case in ("mip", "surfel") else "3dgs"
    fused = case == "same_stream_fused"
    f32 = lambda t: np.ascontiguousarray(t.detach().cpu().numpy(), dtype=np.float32)

    # ---- 1. the scene, on the CPU; and what the activations give in CPU float32 -----------------------------------------
    model = cam = arrays = None
    if a.scene == "B":
        import scenes
        arrays = scenes.scene("B")
        W, H = arrays["W"], arrays["H"]
        for k in ("means3D", "opacities", "colors_precomp", "cov3D_precomp", "viewmatrix", "projmatrix", "campos"):
            out["exp_" + k] = np.ascontiguousarray(arrays[k], dtype=np.float32)
    else:
        if a.scene == "cfg5":  # the scene of DESIGN.md 3.5's open issue
            model, cams, _ = build_config("cfg5", P=40000, K=1, W=240, H=180)
        else:
            model, cams, _ = build_config("cfg1", W=256, H=256)
        cam = cams[0]
        W, H = int(cam.image_width), int(cam.image_height)
        if kind == "surfel":  # two tangent scales
            model = GaussianPointCloud(model._xyz, model._scale[:, :2].contiguous(), model._rot, model._opacity,
                                       model._f_dc, model._f_rest, model.max_sh_degree, model.active_sh_degree)
        if kind == "mip":
            from gaustudio_b200.mip import MipPointCloud
            model = MipPointCloud.from_model(model)
        with torch.no_grad():
            out["exp_means3D"] = f32(model._xyz)
            out["exp_viewmatrix"], out["exp_projmatrix"] = f32(cam.world_view_transform), f32(cam.full_proj_transform)
            out["exp_campos"] = f32(cam.camera_center)
            if fused:  # the forward takes the raw attributes
                out["exp_opacities"], out["exp_scales"], out["exp_rotations"] = (f32(model._opacity), f32(model._scale),
                                                                                 f32(model._rot))
                P_ = model._xyz.shape[0]
                out["exp_f_dc"], out["exp_f_rest"] = f32(model._f_dc.reshape(P_, -1, 3)), f32(model._f_rest.reshape(P_, -1, 3))
            else:
                out["exp_rotations"], out["exp_shs"] = f32(model.get_attribute("rot")), f32(model.get_features)
                rounded = ["rotations"]
                if kind != "mip":  # the Mip renderer's scales and opacities carry the 3D filter, computed on the device
                    out["exp_opacities"], out["exp_scales"] = f32(model.get_attribute("opacity")), f32(model.get_attribute("scale"))
                    rounded += ["opacities", "scales"]

    # ---- 2. CUDA starts here: produce the inputs as the case prescribes and render at once ----------------------------
    dev = torch.device("cuda")
    rec = Recorder(_C, "rasterize_surfels" if kind == "surfel" else "rasterize_gaussians")
    name = {"3dgs": "vanilla_renderer", "mip": "mip_renderer", "surfel": "surfel_renderer"}[kind]
    conf = {"name": name}
    if kind == "3dgs":
        conf["fused_activations"] = fused
    r = renderers.make(conf)
    render_stream = torch.cuda.Stream() if case == "non_default_stream" else None
    scope = torch.cuda.stream(render_stream) if render_stream is not None else contextlib.nullcontext()
    h0 = _C.speculation_stats()
    with scope, torch.no_grad():
        if arrays is not None:
            from gaustudio_b200.rasterizer import GaussianRasterizationSettings, GaussianRasterizer
            t = {k: torch.as_tensor(arrays[k]).to(dev) for k in ("means3D", "opacities", "colors_precomp", "cov3D_precomp",
                                                                  "viewmatrix", "projmatrix", "campos")}
            rs = GaussianRasterizationSettings(H, W, arrays["tanfovx"], arrays["tanfovy"], torch.as_tensor(arrays["bg"]),
                                               arrays["scale_modifier"], t["viewmatrix"], t["projmatrix"], arrays["D"],
                                               t["campos"], False, False)
            GaussianRasterizer(rs)(t["means3D"], torch.zeros_like(t["means3D"]), t["opacities"],
                                   colors_precomp=t["colors_precomp"], cov3D_precomp=t["cov3D_precomp"])
        elif case == "materialised":  # the control: inputs made, the device drained, then the forward
            model.to(dev)
            cam = cam.to(dev)
            props = r.get_gaussians_properties(cam, model)
            torch.cuda.synchronize()
            r.rasterize(cam, model, props=props)
        elif case == "side_stream_waited":  # inputs on a second stream, the render stream waits for it
            side = torch.cuda.Stream()
            with torch.cuda.stream(side):
                model.to(dev)
                cam = cam.to(dev)
                props = r.get_gaussians_properties(cam, model)
            torch.cuda.current_stream().wait_stream(side)
            r.rasterize(cam, model, props=props)
        else:
            model.to(dev)
            if kind == "mip":
                model.compute_3D_filter([cam])
            if case == "after_allocator_churn":
                # blocks of the sizes the forward will ask for, filled with 0xFF (NaN as floats) by kernels queued behind
                # a long-running one, and freed without synchronising: the forward's torch.empty recycles them
                L = _lib.lib()
                P_ = model._xyz.shape[0]
                busy = torch.ones(1 << 26, device=dev)
                for _ in range(8):
                    busy.mul_(1.0000001)
                sizes = [L.gsr_geometry_bytes(P_), L.gsr_image_bytes(W, H), L.gsr_binning_bytes(1 << 20),
                         L.gsr_binning_bytes(2 << 20), 8 * H * W * 4, P_ * 4]
                junk = [torch.empty(int(n), dtype=torch.uint8, device=dev).fill_(0xFF) for n in sizes]
                del junk
            r.render(cam.to(dev), model)

        # ---- 3. the first forward's state, exported before anything else happens -------------------------------------
        args, kw, res = rec.calls[0]
        h1 = _C.speculation_stats()
        if kind == "surfel":
            R, color, radii, allmap, gb, bb, ib = res
            keep = [dict(planes=torch.cat([color, allmap]).clone(), radii=radii.clone(), R=R)]
        else:
            R, color, depth, median, opac, radii, gb, bb, ib = res
            P_ = radii.numel()
            ex = _C.debug_export(P_, W, H, R, gb, bb, ib)
            keep = [dict(ex, planes=torch.cat([color, depth, median, opac]).clone(), radii=radii.clone(), R=R)]

        # ---- 4. only now: synchronise, download the inputs, render twice more from the same device tensors ------------
        torch.cuda.synchronize()
        names = SURFEL_ARG_NAMES if kind == "surfel" else ARG_NAMES
        given = dict(zip(names, args))
        if kw.get("_fused") is not None:
            given["f_dc"], given["f_rest"] = kw["_fused"]
        for k, v in given.items():
            if torch.is_tensor(v):
                out["in_" + k] = f32(v) if v.numel() else np.zeros(0, np.float32)
                out["in_" + k + "_device"] = np.array(v.is_cuda)
            elif v is not None:
                out["in_" + k] = np.array(v)
        out["kernel_size"] = np.array(-1.0 if kw.get("_kernel_size") is None else kw["_kernel_size"])
        stats = [h0, h1]
        for plain in (False, True):
            prev = _C.set_speculation(False) if plain else None
            try:
                res = rec.orig(*args, **kw)
            finally:
                if plain:
                    _C.set_speculation(prev)
            stats.append(_C.speculation_stats())
            if kind == "surfel":
                R, color, radii, allmap, gb, bb, ib = res
                keep.append(dict(planes=torch.cat([color, allmap]), radii=radii, R=R))
            else:
                R, color, depth, median, opac, radii, gb, bb, ib = res
                ex = _C.debug_export(radii.numel(), W, H, R, gb, bb, ib)
                keep.append(dict(ex, planes=torch.cat([color, depth, median, opac]), radii=radii, R=R))
        torch.cuda.synchronize()

    # ---- 5. everything to the npz ---------------------------------------------------------------------------------------
    for i, st in enumerate(keep, 1):
        for k, v in st.items():
            out[f"r{i}_{k}"] = v.cpu().numpy() if torch.is_tensor(v) else np.array(v)
    out["spec_stats"] = np.array(stats, np.int64)  # (hits, redos) before render 1 and after renders 1, 2, 3
    out["case"], out["scene"], out["kind"], out["fused"] = np.array(case), np.array(a.scene), np.array(kind), np.array(fused)
    out["W"], out["H"], out["rounded"] = np.array(W), np.array(H), np.array(rounded, dtype="U16")
    out["module_loading"] = np.array(os.environ.get("CUDA_MODULE_LOADING", ""))
    np.savez(a.out, **out)


if __name__ == "__main__":
    main()
