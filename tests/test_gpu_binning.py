"""-m gpu: the binning (tile scan, two-level scatter, per-tile sort) against a torch restatement of its contract.

Every (Gaussian, binned tile) pair becomes the entry (depth bits << 32 | index); a tile's range is the exclusive prefix
of the per-tile counts; a tile whose range does not fit the binning capacity renders nothing (empty range, no entries);
within a range the entries are in ascending order and the list holds their Gaussian indices.  The binned tiles of a
Gaussian are the bits of its tile mask for rects of up to 32 tiles and the whole rect otherwise.

The restatement reads the rect, tile mask and depth key the projection left in the geometry buffer (the carve of
`carve_geom` in gsr_api.cu, replicated in `geom_fields` and checked against `debug_export`), so it checks the binning
alone: `ranges` and `point_list` must be equal, not close.  Scenes cover a 1x1 image, sizes that are not a multiple of
the 128-pixel super-tile, an image of more than one scan round, rects larger than the image, one tile holding every
Gaussian, super-tiles whose lists expand beyond one shared-memory stage, P = 0 and 1, a pipelined capacity that drops
tiles, a CUDA-graph replay and a bit-identical repeat."""
import math

import numpy as np
import pytest
import torch

import scenes
from test_gpu_foreign_state import Inputs, Run

pytestmark = pytest.mark.gpu


def ball(P, W, H, s0=0.05, seed=0, radius=1.0, pos=(2.2, 1.4, 1.6), opacity=None):
    """P Gaussians in a ball of `radius` at the origin, seen from `pos` (the format of scenes.scene)."""
    rng = np.random.RandomState(seed)
    d = rng.randn(P, 3)
    d /= np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-12)
    xyz = d * (radius * rng.rand(P, 1) ** (1 / 3))
    scales = np.exp(math.log(s0) + 0.5 * rng.randn(P, 3))
    rot = rng.randn(P, 4)
    rot /= np.linalg.norm(rot, axis=1, keepdims=True)
    opac = 1 / (1 + np.exp(-2.0 * rng.randn(P, 1))) if opacity is None else np.full((P, 1), opacity)
    shs = np.concatenate([rng.randn(P, 1, 3), 0.2 * rng.randn(P, 15, 3)], axis=1)
    cam = scenes.camera(W, H, pos=pos)
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    return dict(case="binning", W=W, H=H, D=3, scale_modifier=1.0, bg=np.zeros(3, np.float32), means3D=f32(xyz),
                scales=f32(scales), rotations=f32(rot), opacities=f32(opac), shs=f32(shs),
                viewmatrix=cam.world_view_transform.numpy(), projmatrix=cam.full_proj_transform.numpy(),
                campos=cam.camera_center.numpy(), tanfovx=math.tan(cam.FoVx * 0.5), tanfovy=math.tan(cam.FoVy * 0.5))


def geom_fields(gb, P, with_splat=False):
    """(rect [P,2] uint32 as int64, tile_mask [P], depth [P] float32, tiles_touched [P]) from a geometry buffer, and
    with with_splat=True the whole splat record [P,12] (px, py, A, B, C, o, depth, r, g, b, index bits, tau) after them:
    carve_geom's layout, every array at the next 256-byte boundary (splat [P][3] float4, rect [P] uint2, cov3D [P][6],
    clamped [P] u8, radii, tiles_touched, tile_mask [P] u32)."""
    base = (-gb.data_ptr()) % 256
    offs, p = {}, base
    for name, nbytes in (("splat", 48), ("rect", 8), ("cov3D", 24), ("clamped", 1), ("radii", 4), ("touched", 4),
                         ("mask", 4)):
        p = (p + 255) // 256 * 256
        offs[name] = p
        p += nbytes * P
    view = lambda name, n, dt: gb[offs[name]:offs[name] + n * P].view(dt)
    rect = view("rect", 8, torch.int32).view(P, 2).long() & 0xffffffff
    mask = view("mask", 4, torch.int32).long() & 0xffffffff
    splat = view("splat", 48, torch.float32).view(P, 12)
    touched = view("touched", 4, torch.int32).long()
    if with_splat:
        return rect, mask, splat[:, 6].contiguous(), touched, splat
    return rect, mask, splat[:, 6].contiguous(), touched


def reference_binning(rect, mask, depth, W, H, cap=None):
    """-> (ranges [T,2] int64, point_list [binned] int64) of the binning contract (module docstring)."""
    dev = rect.device
    P = rect.shape[0]
    gx, gy = (W + 15) // 16, (H + 15) // 16
    T = gx * gy
    x0, x1 = rect[:, 0] & 0xffff, rect[:, 0] >> 16
    y0, y1 = rect[:, 1] & 0xffff, rect[:, 1] >> 16
    w = (x1 - x0).clamp(min=0)
    n = w * (y1 - y0).clamp(min=0)
    idx = torch.arange(P, device=dev)
    # rects of <= 32 tiles: the set bits of the mask
    small = (n > 0) & (n <= 32)
    bit = torch.arange(32, device=dev)
    on = small[:, None] & (bit[None] < n[:, None]) & (((mask[:, None] >> bit[None]) & 1) == 1)
    g_s, b_s = on.nonzero(as_tuple=True)
    ws = w[g_s].clamp(min=1)
    t_s = (y0[g_s] + b_s // ws) * gx + x0[g_s] + b_s % ws
    # larger rects: every tile
    big = (n > 32).nonzero(as_tuple=True)[0]
    nb = n[big]
    g_b = torch.repeat_interleave(big, nb)
    first = torch.repeat_interleave(torch.cumsum(nb, 0) - nb, nb)
    i_b = torch.arange(g_b.numel(), device=dev) - first
    wb = w[g_b]
    t_b = (y0[g_b] + i_b // wb) * gx + x0[g_b] + i_b % wb
    g_all, t_all = torch.cat([g_s, g_b]), torch.cat([t_s, t_b])
    dbits = depth.view(torch.int32).long() & 0xffffffff
    key = (dbits[g_all] << 32) | idx[g_all]
    order = torch.sort(key, stable=True).indices
    order = order[torch.sort(t_all[order], stable=True).indices]
    count = torch.bincount(t_all, minlength=T)
    start = torch.cumsum(count, 0) - count
    fits = torch.ones_like(count, dtype=torch.bool) if cap is None else start + count <= cap
    live = (count > 0) & fits
    ranges = torch.where(live[:, None], torch.stack([start, start + count], 1), torch.zeros(T, 2, dtype=torch.long, device=dev))
    keep = fits[t_all[order]]
    return ranges, g_all[order][keep]


def check(run, cap=None):
    """The export of `run` equals the restatement built from its own geometry buffer; -> the export."""
    inp = run.inp
    ex = run.export()
    rect, mask, depth, touched = geom_fields(run.gb, inp.P)
    vis = ex["depths"] != 0
    assert torch.equal(depth.cpu()[vis], ex["depths"][vis]), "geometry carve replica disagrees with debug_export"
    assert torch.equal(touched.cpu().int(), ex["tiles_touched"]), "geometry carve replica disagrees with debug_export"
    ranges, pl = reference_binning(rect, mask, depth, inp.W, inp.H, cap)
    assert torch.equal(ex["ranges"].long(), ranges.cpu()), "tile ranges differ"
    assert torch.equal(ex["point_list"].long(), pl.cpu()), "point list differs"
    return ex


def _run(s, cap=0):
    return Run(Inputs(s, torch.device("cuda")), "zero", cap=cap)


def one_big(W, H, extra=0, seed=1):
    """A Gaussian at the origin whose rect covers the whole image, and `extra` small ones."""
    s = ball(1 + extra, W, H, s0=0.02, seed=seed)
    s["means3D"][0] = 0.0
    s["scales"][0] = 3.0
    s["opacities"][0] = 0.9
    return s


def one_tile(P, W=300, H=200):
    """P small Gaussians projecting into the image's centre tile."""
    return ball(P, W, H, s0=0.002, seed=3, radius=0.004)


def many_big(P, W=300, H=200):
    """P Gaussians with rects of more than 32 tiles: every super-tile list expands to tens of tiles per entry."""
    return ball(P, W, H, s0=0.25, seed=4, radius=0.3, opacity=0.5)


SCENES = {
    "1x1": lambda: ball(300, 1, 1, s0=0.1),
    "136x200": lambda: ball(2000, 136, 200),
    "300x77": lambda: ball(2000, 300, 77),
    "1000x530": lambda: ball(20000, 1000, 530, s0=0.03),
    "4096x2304": lambda: ball(60000, 4096, 2304, s0=0.02),
    "8192x4608": lambda: ball(60000, 8192, 4608, s0=0.02),  # 2304 super-tiles: two windows of the coarse histogram
    "one_big": lambda: one_big(300, 200),
    "one_big_mixed": lambda: one_big(1000, 600, extra=3000),
    "one_tile": lambda: one_tile(40000),
    "many_big": lambda: many_big(3000),
    "P1": lambda: one_big(200, 120),
    "P1_small": lambda: ball(1, 64, 64, s0=0.05),
}


@pytest.mark.parametrize("name", list(SCENES))
def test_binning_matches_restatement(name):
    s = SCENES[name]()
    run = _run(s)
    ex = check(run)
    if name.startswith("one_big") or name == "many_big":
        n = ex["tiles_touched"]
        assert int(n.max()) > 32, "no rect took the large-rect path"
    if name == "one_tile":
        rg = ex["ranges"].long()
        assert int((rg[:, 1] - rg[:, 0]).max()) > 20000, "the crowded tile is not crowded"


def test_all_culled_and_empty():
    """P Gaussians all behind the camera bin nothing; P = 0 never reaches the library."""
    from gaustudio_b200 import _C
    s = ball(500, 200, 120)
    s["means3D"] = np.ascontiguousarray(s["means3D"] * 0.01 + 2.0 * np.asarray(s["campos"], np.float32), np.float32)
    run = _run(s)
    ex = check(run)
    assert ex["num_binned"] == 0
    dev = torch.device("cuda")
    z = torch.zeros(0, 3, device=dev)
    out = _C.rasterize_gaussians(torch.zeros(3, device=dev), z, torch.zeros(0, 3, device=dev),
                                 torch.zeros(0, 1, device=dev), torch.zeros(0, 3, device=dev),
                                 torch.zeros(0, 4, device=dev), 1.0, torch.zeros(0, device=dev),
                                 torch.eye(4, device=dev), torch.eye(4, device=dev), 0.5, 0.5, 40, 60,
                                 torch.zeros(0, 16, 3, device=dev), 3, torch.zeros(3, device=dev), False, False)
    assert out[0] == 0 and not out[1].any()


@pytest.mark.parametrize("frac", [0.3, 0.7])
def test_pipelined_capacity_drops_tiles(frac):
    """A fixed capacity below the binned count: the tiles past it have empty ranges, the others are exact."""
    s = ball(20000, 1000, 530, s0=0.03, seed=5)
    full = _run(s)
    cap = int(full.binned * frac)
    run = _run(s, cap=cap)
    ex = check(run, cap=cap)
    rg = ex["ranges"].long()
    assert int((rg[:, 1] > 0).sum()) < int((full.export()["ranges"][:, 1] > 0).sum()), "no tile was dropped"


def test_repeat_is_bit_identical():
    s = ball(20000, 1000, 530, s0=0.03, seed=6)
    a, b = _run(s).export(), _run(s).export()
    for k in ("ranges", "point_list", "n_contrib", "final_T"):
        assert torch.equal(a[k], b[k]), k


def test_graph_replay():
    """The forward captured in a CUDA graph (fixed-capacity mode) bins exactly what the restatement says, replay after
    replay."""
    from gaustudio_b200 import _C
    dev = torch.device("cuda")
    s = ball(20000, 1000, 530, s0=0.03, seed=7)
    inp = Inputs(s, dev)
    t = inp.t
    cap = _run(s).binned + 4096
    state = _C.pipeline_state()
    _C.set_pipelined(True, fixed_capacity=cap)
    try:
        args = lambda: (inp.bg, t["means3D"], t["colors_precomp"], t["opacities"], t["scales"], t["rotations"], 1.0,
                        t["cov3D_precomp"], inp.view, inp.proj, float(s["tanfovx"]), float(s["tanfovy"]), inp.H,
                        inp.W, t["shs"], 3, inp.campos, False, False)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            _C.rasterize_gaussians(*args())
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = _C.rasterize_gaussians(*args())
        exports = []
        for _ in range(2):
            g.replay()
            torch.cuda.synchronize()
            gb, bb, ib = out[6], out[7], out[8]
            ex = _C.debug_export(inp.P, inp.W, inp.H, out[0], gb, bb, ib)
            rect, mask, depth, _ = geom_fields(gb, inp.P)
            ranges, pl = reference_binning(rect, mask, depth, inp.W, inp.H, cap)
            assert torch.equal(ex["ranges"].long(), ranges), "tile ranges differ after replay"
            assert torch.equal(ex["point_list"].long(), pl), "point list differs after replay"
            exports.append(ex["point_list"].clone())
        assert torch.equal(exports[0], exports[1])
    finally:
        _C.restore_pipeline(state)
