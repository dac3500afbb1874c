"""CPU: the float64 culling checks of tests/cull_ref64.py report every seeded fault, the float32 restatement of
tile_mask_of passes them on the edge families (10^5 Gaussians each), and may_touch keeps every 8x4 block and 16x16 tile
a pixel needs on the same families."""
import numpy as np
import pytest

import cull_ref64 as K

N_FAMILY = 100000
IMGS = ("1x1", "17x9", "250x170", "1920x1080", "8192x4608")
TIGHT_SHARE = K.TIGHT_SHARE


def scene(fam, n=N_FAMILY, seed=0, imgs=IMGS, mip=None):
    """n Gaussians of family `fam`, split over the images: -> list of (records, restated mask)."""
    out = []
    for j, img in enumerate(imgs):
        W, H = K.IMAGES[img]
        dil = 0.3 if mip is None else mip
        f = K.family(fam, n // len(imgs), W, H, seed=seed + 17 * j, dil=dil)
        o = f["o"] if mip is None else K.mip_input_opacity(f["cov"], f["o"], mip)  # the family's o after the filter
        r = K.records(f["px"], f["py"], f["cov"], o, W, H, dil=dil, mip=mip is not None)
        out.append((img, r))
    return out


def one(px, py, a, b, c, o, W, H):
    """A hand-placed scene: records of the listed Gaussians (screen-space covariances before the 0.3 dilation)."""
    return K.records(np.asarray(px, float), np.asarray(py, float), (np.asarray(a, float), np.asarray(b, float),
                                                                      np.asarray(c, float)), np.asarray(o, float), W, H)


# ---- seeded faults ----------------------------------------------------------------------------------------------------
def _needles():
    (_, r), = scene("needles", 20000, seed=5, imgs=("250x170",))
    return r


def test_fault_cleared_needed_bit():
    r = _needles()
    m = K.tile_mask_f32(r)
    rep = K.check_mask(r, m)
    assert not rep.failed(), rep.text()
    # clear one bit of a tile a pixel needs, in 50 Gaussians
    n, w, tx, ty, ex = K._bits(r)
    px, py, A, B, C = (np.asarray(r[k], np.float64) for k in ("px", "py", "A", "B", "C"))
    qmin, gmin = K.block_qmin(px, py, A, B, C, tx * 16, ty * 16, 16, 16, r["W"], r["H"])
    req = ex & (gmin <= (2 * np.log(255 * np.asarray(r["o"], np.float64)) + K.SLACK_ABS)[:, None]) & (n <= 32)[:, None]
    rows = np.nonzero(req.any(1))[0][:50]
    assert len(rows) == 50
    bad = m.copy()
    for i in rows:
        bad[i] &= ~(1 << int(np.nonzero(req[i])[0][-1]))
    assert K.check_mask(r, bad).failed() == {"coverage"}
    # one bit is enough
    one_bad = m.copy()
    one_bad[rows[0]] &= ~(1 << int(np.nonzero(req[rows[0]])[0][0]))
    assert K.check_mask(r, one_bad).failed() == {"coverage"}


def test_fault_bit_beyond_rect():
    r = _needles()
    m = K.tile_mask_f32(r)
    n = (r["x1"] - r["x0"]) * (r["y1"] - r["y0"])
    i = int(np.nonzero((n > 0) & (n < 32))[0][0])
    bad = m.copy()
    bad[i] |= 1 << int(n[i])
    assert "shape" in K.check_mask(r, bad).failed()


def test_fault_all_margins_removed():
    """Gaussians whose only pixel in a tile sits just outside q = tau (q = tau + 5e-5, inside the check's slack): the
    restatement without its margins drops that tile, with them it keeps it.  Round splats with o = 1, the pixel at the
    first or the last column of a tile; the conic is set from the float32 centre so that q lands where it should.

    The margin this fault takes away is taum's 1e-5 S + 1e-3: the x-extent's 1.0001 and 0.01 px alone would still keep
    the tile (0.01 px is worth ~0.07 in q here), and with taum's margin in place they are not load-bearing in the
    restatement at all: dropping only them leaves every edge family passing
    (test_extent_margins_alone_are_not_load_bearing)."""
    W, H = 250, 64
    tau = float(np.float32(2) * np.log(np.float32(255)))
    cols = 16 * np.arange(2, 14)
    px = np.concatenate([cols - 3.3, cols + 15 + 3.3]).astype(np.float32).astype(np.float64)
    dx = np.concatenate([cols, cols + 15]) - px
    cov = dx * dx / (tau + 5e-5) - 0.3  # A = C = 1 / (cov + 0.3)
    py = np.full(px.shape, 24.0)
    r = one(px, py, cov, np.zeros(px.shape), cov, np.ones(px.shape), W, H)
    good = K.check_mask(r, K.tile_mask_f32(r))
    assert not good.failed(), good.text()
    assert K.check_mask(r, K.tile_mask_f32(r, margins=False)).failed() == {"coverage"}


def test_extent_margins_alone_are_not_load_bearing():
    """The restatement with taum's margin but without the x-extent's 1.0001 / 0.01 px passes coverage on the edge
    families: taum's 1e-5 S + 1e-3 exceeds the float32 rounding of the extent.  (So no seeded fault can show the 0.01
    px margin needed; the kernel keeps it for its FMA-contracted arithmetic, which this restatement does not model.)"""
    for fam in K.FAMILIES:
        for img, r in scene(fam, 10000, seed=41):
            rep = K.check_mask(r, K.tile_mask_f32(r, extent_margins=False))
            assert "coverage" not in rep.failed(), f"{fam} {img}: {rep.text()}"


def test_fault_band_clamp_moved():
    """The row band clamped to H + 15 instead of H - 1: tiles of the last, partial tile row get bits for ellipses that
    only reach the rows below the image."""
    W, H = 17, 9
    py = np.linspace(H + 1.5, 15.5, 40)
    px = np.linspace(2.0, 14.0, 40)
    r = one(px, py, np.full(40, 0.5), np.zeros(40), np.full(40, 0.5), np.full(40, 0.9), W, H)
    assert not K.check_mask(r, K.tile_mask_f32(r)).failed()
    assert K.check_mask(r, K.tile_mask_f32(r, hclamp=H + 15)).failed() == {"tightness"}
    for fam in ("partial", "needles"):
        (_, r), = scene(fam, 20000, seed=9, imgs=("17x9",))
        assert K.check_mask(r, K.tile_mask_f32(r, hclamp=H + 15)).failed() == {"tightness"}, fam


def test_fault_all_ones():
    """'keep everything' passes coverage and shape but not tightness."""
    r = _needles()
    n = (r["x1"] - r["x0"]) * (r["y1"] - r["y0"])
    allm = np.where(n >= 32, 0xffffffff, (np.int64(1) << np.minimum(n, 32)) - 1)
    allm = np.where(r["o"] < K.O_CUT, 0, allm)
    assert K.check_mask(r, allm).failed() == {"tightness"}


def test_fault_dead_opacity_and_guard():
    """A bit for o < 0.0039, and a partial mask where the guard must keep everything, are shape faults."""
    W, H = 250, 170
    r = one([100.5, 100.5], [80.0, 80.0], [0.7, 4.0], [0.0, 5.0], [0.7, 4.0], [0.00389, 0.5], W, H)
    m = K.tile_mask_f32(r)
    assert m[0] == 0 and K.check_mask(r, m).failed() == set()
    bad = m.copy()
    bad[0] = 1
    assert K.check_mask(r, bad).failed() == {"shape"}
    assert np.float64(r["A"][1]) * r["C"][1] - np.float64(r["B"][1]) ** 2 < 0  # indefinite conic: the guard fires
    bad = m.copy()
    bad[1] = 1
    assert K.check_mask(r, bad).failed() == {"shape"}


# ---- the restatement on the edge families -----------------------------------------------------------------------------
@pytest.mark.parametrize("fam", K.FAMILIES)
def test_restatement_passes_on_edge_family(fam):
    set_, loose = 0, 0
    stats = []
    for img, r in scene(fam):
        rep = K.check_mask(r, K.tile_mask_f32(r))
        assert not rep.failed(), f"{fam} {img}: {rep.text()}"
        st = rep.stats
        set_ += st["set"]
        loose += st["tight_share"] * st["set"]
        stats.append((img, st["masked"], st["slack_min"], st["worst_tight"], st["fallback"]))
    share = loose / max(set_, 1)
    print(f"\n{fam}: tightness share {share:.4f}; (image, masked, worst slack, worst box/taum, fallback) {stats}")
    assert share <= TIGHT_SHARE[fam], share
    assert sum(s[1] for s in stats) > N_FAMILY // 10


@pytest.mark.parametrize("k", [0.0, 0.1, 0.3])
def test_restatement_passes_on_mip_families(k):
    """The Mip filter: cov + k I and opacity o coef, o placed across 0.0039 after the filter.  At k = 0 the tightness
    share stays within MIP0_TIGHT_SHARE, and most degenerate covariances are dead (coef 0: opacity exactly 0); the
    others are those whose float32 det0 rounds above 1e-6, and reach the mask with a near-singular conic."""
    for fam in ("needles", "opacity", "degenerate", "boundaries"):
        set_, loose = 0, 0.0
        for img, r in scene(fam, 20000, seed=31, mip=k):
            rep = K.check_mask(r, K.tile_mask_f32(r))
            assert not rep.failed(), f"{fam} {img} k={k}: {rep.text()}"
            set_ += rep.stats["set"]
            loose += rep.stats["tight_share"] * rep.stats["set"]
            if fam == "degenerate" and k == 0.0:
                live = (r["x1"] - r["x0"]) * (r["y1"] - r["y0"]) > 0
                assert (r["o"][live] == 0).mean() >= 0.5, (r["o"][live] == 0).mean()
        if k == 0.0 and fam != "degenerate":
            assert loose / max(set_, 1) <= K.MIP0_TIGHT_SHARE[fam], (fam, loose / set_)


def test_families_reach_their_edges():
    """What each family is there for: 32- and 33-tile rects of every shape, strips of <= 32 tiles, o on both sides of
    the cut, B = 0 and 45-degree needles, and the guard firing."""
    shapes = set()
    for img, r in scene("rect32"):
        w, h = r["x1"] - r["x0"], r["y1"] - r["y0"]
        shapes |= set(zip(w.tolist(), h.tolist()))
    assert {(4, 8), (8, 4), (32, 1), (1, 32), (33, 1)} <= shapes
    n_strip = 0
    for _, r in scene("strips", 20000):
        n = (r["x1"] - r["x0"]) * (r["y1"] - r["y0"])
        far = (r["px"] < -1000) | (r["px"] > r["W"] + 1000) | (r["py"] < -1000) | (r["py"] > r["H"] + 1000)
        n_strip += int(((n > 0) & (n <= 32) & far).sum())
    assert n_strip > 1000
    o = np.concatenate([r["o"] for _, r in scene("opacity", 20000)])
    assert (o < K.O_CUT).sum() > 100 and ((o >= K.O_CUT) & (o < np.float32(1 / 255))).sum() > 100
    assert (o == np.float32(1 / 255)).sum() > 100
    B = np.concatenate([r["B"] for _, r in scene("needles", 20000)])
    assert (B == 0).sum() > 100
    deg = scene("degenerate", 20000)
    assert sum(K.check_mask(r, K.tile_mask_f32(r)).stats["fallback"] for _, r in deg) > 1000


# ---- may_touch, widened -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bw,bh", [(8, 4), (16, 16)])
@pytest.mark.parametrize("fam", K.FAMILIES)
def test_cull_bound_is_conservative_on_edge_families(fam, bw, bh):
    """test_oracle_props.test_cull_bound_is_conservative on the edge families: may_touch never drops a block with a
    pixel at q <= tau + 1e-4 + 1e-6 S."""
    need, miss = 0, 0
    for img, r in scene(fam, 50000, seed=3):
        m, share, nd = K.check_may_touch(r, bw, bh, K=16, seed=len(img))
        miss += m
        need += nd
    print(f"\n{fam} {bw}x{bh}: {need} blocks needed")
    assert miss == 0, miss
    assert need > 1000
