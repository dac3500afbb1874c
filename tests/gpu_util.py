import hashlib

import numpy as np
import torch


def array_digest(a):
    """SHA-1 of an array's dtype, shape and bytes."""
    a = np.ascontiguousarray(a)
    return hashlib.sha1(f"{a.dtype.str}{a.shape}".encode() + a.tobytes()).hexdigest()


def assert_scene_matches_fixture(s, G):
    """The scene generator still produces the input arrays a ref_case fixture was made from (stored as digests)."""
    for k, v in s.items():
        if isinstance(v, np.ndarray):
            assert array_digest(v) == str(G["insha_" + k]), f"scene generator drifted from the fixture ({k})"


def new_rasterize(rs, means3D, means2D, opacities, **kw):
    from gaustudio_b200.rasterizer import GaussianRasterizer
    return GaussianRasterizer(rs)(means3D, means2D, opacities, **kw)


def ref_rasterize(rs, means3D, means2D, opacities, **kw):
    from oracle import ref_driver
    return ref_driver.rasterize(rs, means3D, means2D, opacities, **kw)


def oracle_run(s):
    """CPU oracle outputs + grads in the naming of scenes.run_torch."""
    from oracle.oracle import Oracle
    o = Oracle()
    out = o.forward(s["means3D"], s["opacities"], s["viewmatrix"], s["projmatrix"], s["campos"], s["tanfovx"],
                    s["tanfovy"], s["W"], s["H"], s["D"], shs=s.get("shs"), colors_precomp=s.get("colors_precomp"),
                    scales=s.get("scales"), rotations=s.get("rotations"), cov3D_precomp=s.get("cov3D_precomp"),
                    scale_modifier=s["scale_modifier"])
    g = o.backward(s["dL_color"], s["dL_depth"][0], s["dL_median"], s["dL_opacity"][0], bg=s["bg"])
    r = dict(color=out["color"], radii=out["radii"], depth=out["depth"], median=out["median"], opacity=out["opacity"],
             num_rendered=out["num_rendered"], g_means2D=g["means2D"], g_means3D=g["means3D"],
             g_opacities=g["opacities"])
    if "shs" in s:
        r["g_shs"] = g["shs"]
    else:
        r["g_colors_precomp"] = g["colors_precomp"]
    if "scales" in s:
        r["g_scales"], r["g_rotations"] = g["scales"], g["rotations"]
    else:
        r["g_cov3D_precomp"] = g["cov3D_precomp"]
    return r


def assert_grads_close(a, b, rel=1e-3, floor=1e-4, what="", scale=None):
    """BASELINE: <= 1e-3 relative on gradients, with an absolute floor (relative to the tensor's scale)
    because the reference's float atomics make its own gradients order-dependent.  scale: the largest magnitude of the
    whole reference tensor when a and b are samples of it."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    scale = np.abs(b).max() if scale is None else scale
    err = np.abs(a - b)
    bound = rel * np.abs(b) + floor * scale + 1e-30
    bad = err > bound
    assert not bad.any(), f"{what}: {int(bad.sum())}/{bad.size} beyond tolerance, worst {err.max():.3e} (scale {scale:.3e})"


def assert_images_close(a, b, atol=1e-4, outlier_frac=0.0, what=""):
    err = np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64))
    frac = (err > atol).mean()
    assert frac <= outlier_frac, f"{what}: {frac:.2e} of pixels beyond {atol} (max {err.max():.3e})"


def reference_tile_segments(point_list, ranges, T, n_crowded, n_random, seed, extra=()):
    """A fixed selection of tiles of the reference's sorted list (the n_crowded most crowded ones, the tiles `extra` and
    n_random other non-empty ones) with their segments of the list: {seg_tiles, seg_ranges, seg_list}, seg_ranges
    indexing seg_list."""
    rg = np.asarray(ranges.cpu() if torch.is_tensor(ranges) else ranges).astype(np.int64).reshape(-1, 2)[:T]
    pl = np.asarray(point_list.cpu() if torch.is_tensor(point_list) else point_list)
    n = rg[:, 1] - rg[:, 0]
    crowded = np.union1d(np.argsort(-n, kind="stable")[:n_crowded], np.asarray(extra, np.int64))
    rest = np.setdiff1d(np.nonzero(n)[0], crowded)
    tiles = np.sort(np.concatenate([crowded, np.random.RandomState(seed).choice(rest, n_random, replace=False)]))
    segs = [pl[rg[t, 0]:rg[t, 1]] for t in tiles]
    ends = np.cumsum([len(x) for x in segs])
    return {"seg_tiles": tiles.astype(np.int64), "seg_ranges": np.stack([ends - n[tiles], ends], 1).astype(np.int64),
            "seg_list": np.concatenate(segs).astype(np.int32)}


def assert_binned_list_is_culled_reference_list(ex, ref_point_list, ref_ranges, W, H, P, tiles=None):
    """The binning keeps a (Gaussian, tile) pair of the reference's rect only if the Gaussian can reach alpha >= 1/255 on
    some pixel of the tile (exact tile culling).  So the sorted list must be the REFERENCE's sorted list with entries
    removed -- same relative order -- and every removed entry must be provably inert: no pixel of its tile passes the
    reference's own `power <= 0 && alpha >= 1/255` test (forward.cu:349-355).  Returns the number of removed entries.
    ex: _C.debug_export dict; ref_point_list [R_ref], ref_ranges [>=T, 2]: the reference's (or the pinned oracle's).
    tiles: check only these tiles; ref_point_list / ref_ranges then hold their segments only (reference_tile_segments)."""
    dev = ex["point_list"].device
    our_pl, our_rg = ex["point_list"].long(), ex["ranges"].long()
    T = our_rg.shape[0]
    if tiles is None:
        tiles = torch.arange(T, device=dev)
        assert our_pl.numel() == ex["num_binned"]
    else:
        tiles = torch.as_tensor(np.asarray(tiles, np.int64)).to(dev)
        our_rg = our_rg[tiles]
        our_pl = torch.cat([our_pl[int(a):int(b)] for a, b in our_rg.tolist()])
    ref_pl = torch.as_tensor(np.asarray(ref_point_list.cpu() if torch.is_tensor(ref_point_list) else ref_point_list).astype(np.int64)).to(dev)
    ref_rg = torch.as_tensor(np.asarray(ref_ranges.cpu() if torch.is_tensor(ref_ranges) else ref_ranges).astype(np.int64)).to(dev).reshape(-1, 2)[:tiles.numel()]
    ref_tile = torch.repeat_interleave(tiles, ref_rg[:, 1] - ref_rg[:, 0])
    our_tile = torch.repeat_interleave(tiles, our_rg[:, 1] - our_rg[:, 0])
    assert ref_tile.numel() == ref_pl.numel(), "reference ranges do not cover its list"
    assert our_tile.numel() == our_pl.numel()
    ref_key, our_key = ref_tile * P + ref_pl, our_tile * P + our_pl
    kept = torch.isin(ref_key, our_key)
    assert int(kept.sum()) == our_key.numel(), "binned an instance the reference does not have"
    assert torch.equal(ref_key[kept], our_key), "binned list is not the reference's order"
    dt, dg = ref_tile[~kept], ref_pl[~kept]
    gx = (W + 15) // 16
    px0, py0 = ((dt % gx) * 16).float(), ((dt // gx) * 16).float()
    m2, co = ex["means2D"][dg], ex["conic_opacity"][dg]
    off = torch.arange(16, device=dev, dtype=torch.float32)
    step = 1 << 16
    for c in range(0, dg.numel(), step):
        sl = slice(c, c + step)
        X, Y = px0[sl, None, None] + off[None, None, :], py0[sl, None, None] + off[None, :, None]
        dx, dy = m2[sl, 0, None, None] - X, m2[sl, 1, None, None] - Y
        A, B, C, o = (co[sl, i, None, None] for i in range(4))
        power = -0.5 * (A * dx * dx + C * dy * dy) - B * dx * dy
        alpha = torch.clamp(o * torch.exp(power), max=0.99)
        live = (X < W) & (Y < H) & (power <= 0) & (alpha >= 1.0 / 255.0)
        assert not bool(live.any()), "a culled (Gaussian, tile) pair could have contributed"
    return int((~kept).sum())
