"""The debug snapshot of the three rasterizer modules (gaustudio's `raster_settings.debug`): when a forward or backward
call fails, a CPU copy of its arguments is written to snapshot_fw.dump / snapshot_bw.dump in the working directory and
a fixed message is printed before the exception propagates.  No GPU needed: a forward on CPU tensors fails before any
device work, and the backward's native call is replaced by one that fails."""
import types

import pytest
import torch

from gaustudio_b200 import _C, mip_rasterizer, rasterizer, surfel_rasterizer

FW = "\nAn error occured in forward. Please forward snapshot_fw.dump for debugging.\n"
BW_3DGS = "\nAn error occured in backward. Writing snapshot_bw.dump for debugging.\n\n"
BW_SURFEL = "\nAn error occured in backward. Please forward snapshot_bw.dump for debugging.\n"

P, H, W = 4, 8, 8


def _settings(module):
    fields = dict(image_height=H, image_width=W, tanfovx=0.5, tanfovy=0.5, bg=torch.zeros(3), scale_modifier=1.0,
                  viewmatrix=torch.eye(4), projmatrix=torch.eye(4), sh_degree=0, campos=torch.zeros(3),
                  prefiltered=False, debug=True)
    if "kernel_size" in module.GaussianRasterizationSettings._fields:
        fields["kernel_size"] = 0.1
    return module.GaussianRasterizationSettings(**fields)


def _inputs(module):
    g = torch.Generator().manual_seed(0)
    scales = torch.rand(P, 2 if module is surfel_rasterizer else 3, generator=g)
    return dict(means3D=torch.rand(P, 3, generator=g), means2D=torch.zeros(P, 3), opacities=torch.rand(P, 1, generator=g),
                shs=torch.rand(P, 1, 3, generator=g), scales=scales, rotations=torch.rand(P, 4, generator=g))


@pytest.mark.parametrize("module", [rasterizer, mip_rasterizer, surfel_rasterizer], ids=["3dgs", "mip", "surfel"])
def test_forward_failure_writes_snapshot_and_prints_message(module, tmp_path, monkeypatch, capsys):
    monkeypatch.chdir(tmp_path)
    inputs = _inputs(module)
    with pytest.raises(RuntimeError, match="CUDA"):
        module.GaussianRasterizer(_settings(module))(**inputs)
    assert capsys.readouterr().out == FW
    assert sorted(p.name for p in tmp_path.iterdir()) == ["snapshot_fw.dump"]
    snapshot = torch.load(tmp_path / "snapshot_fw.dump")
    assert torch.equal(snapshot[1], inputs["means3D"]) and torch.equal(snapshot[3], inputs["opacities"])
    if module is mip_rasterizer:
        assert snapshot[-1] == 0.1  # kernel_size


@pytest.mark.parametrize("module,native,message", [
    (rasterizer, "rasterize_gaussians_backward", BW_3DGS),
    (mip_rasterizer, "rasterize_gaussians_mip_backward", BW_3DGS),
    (surfel_rasterizer, "rasterize_surfels_backward", BW_SURFEL)], ids=["3dgs", "mip", "surfel"])
def test_backward_failure_writes_snapshot_and_prints_message(module, native, message, tmp_path, monkeypatch, capsys):
    monkeypatch.chdir(tmp_path)

    def fail(*args):
        raise RuntimeError("native backward failed")
    monkeypatch.setattr(_C, native, fail)
    x = _inputs(module)
    e, radii, buf = torch.empty(0), torch.ones(P, dtype=torch.int32), torch.zeros(16, dtype=torch.uint8)
    if module is surfel_rasterizer:
        saved = (e, x["means3D"], x["scales"], x["rotations"], radii, x["shs"], buf, buf, buf)
        grads = (torch.zeros(3, H, W), None, torch.zeros(9, H, W))
        function = surfel_rasterizer._RasterizeGaussians
    else:
        saved = (e, x["means3D"], x["scales"], x["rotations"], e, radii, x["shs"], buf, buf, buf)
        if module is mip_rasterizer:
            saved += (x["opacities"],)
        grads = (torch.zeros(3, H, W), None, torch.zeros(1, H, W), torch.zeros(3, H, W), torch.zeros(1, H, W))
        function = rasterizer._RasterizeGaussians
    ctx = types.SimpleNamespace(raster_settings=_settings(module), num_rendered=0, saved_tensors=saved)
    with pytest.raises(RuntimeError, match="native backward failed"):
        function.backward(ctx, *grads)
    assert capsys.readouterr().out == message
    assert sorted(p.name for p in tmp_path.iterdir()) == ["snapshot_bw.dump"]
    snapshot = torch.load(tmp_path / "snapshot_bw.dump")
    assert torch.equal(snapshot[1], x["means3D"])
    if module is mip_rasterizer:
        assert torch.equal(snapshot[4], x["opacities"]) and snapshot[-1] == 0.1
