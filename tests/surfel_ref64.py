"""Float64 torch restatement of the surfel rasterizer's contract (DESIGN.md §3, surfel rasterizer; include/gsr.h,
gsr_surfel_forward).

Dense over (pixel, Gaussian): every pixel tests every Gaussian's tile rect, Gaussians are composited front to back in
(float32 view depth, index) order with the contract's thresholds.  Everything downstream of the discrete decisions is
differentiable by autograd, which makes this the gradient reference of gsr_surfel_backward (the 0.99 clamp passes no
gradient, the normal's camera-facing flip is held constant, the median depth follows the median splat's z).

Ambiguity flags (like comp_ref64): a pixel is flagged when one of its decisions lies within float32 rounding of the
threshold -- alpha vs 1/255, T(1-alpha) vs 1e-4, T vs 0.5, rho3 vs rho2, z vs 0.2, o G vs the 0.99 clamp -- or when a
Gaussian's tile rect edge (or its integer radius) is within rounding of a tile boundary there.  Flagged pixels are
left out of comparisons and their upstream gradients are zeroed.
"""
import math

import torch

NEAR, FAR = 0.2, 100.0
REL = 2e-3  # relative rounding band of the alpha / transmittance decisions (float32 ray-splat arithmetic, see below)


def rotmat(q):
    """[P,3,3] rotation matrices (row, col) of quaternions (w, x, y, z); not normalised."""
    w, x, y, z = q.unbind(-1)
    return torch.stack([
        torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
        torch.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
        torch.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def sh_colors(shs, D, means, campos):
    from gaustudio_b200.renderers.vanilla_renderer import eval_sh
    d = means - campos[None]
    d = d / d.norm(dim=1, keepdim=True)
    return torch.clamp(eval_sh(D, shs.transpose(1, 2), d) + 0.5, min=0.0)


def project(means, scales, rots, view, proj, W, H, mod=1.0, delta=None):
    """Per-Gaussian geometry.  delta [P,2]: the screen-space translation of the means2D statistic (Tu += dx Tw,
    Tv += dy Tw; mean2D follows)."""
    P = means.shape[0]
    hom = torch.cat([means, torch.ones_like(means[:, :1])], 1)
    pv = hom @ view[:, :3]
    R = rotmat(rots)
    tu = R[:, :, 0] * scales[:, 0:1] * mod
    tv = R[:, :, 1] * scales[:, 1:2] * mod
    cu, cv, cp = tu @ proj[:3], tv @ proj[:3], hom @ proj
    hx = lambda c: W / 2 * c[:, 0] + (W - 1) / 2 * c[:, 3]
    hy = lambda c: H / 2 * c[:, 1] + (H - 1) / 2 * c[:, 3]
    Tu = torch.stack([hx(cu), hx(cv), hx(cp)], 1)
    Tv = torch.stack([hy(cu), hy(cv), hy(cp)], 1)
    Tw = torch.stack([cu[:, 3], cv[:, 3], cp[:, 3]], 1)
    if delta is not None:
        Tu = Tu + delta[:, 0:1] * Tw
        Tv = Tv + delta[:, 1:2] * Tw
    nr = R[:, :, 2] @ view[:3, :3]
    facing = (nr * pv).sum(1).detach()
    sign = torch.where(facing > 0, -1.0, 1.0).to(nr.dtype)
    nv = nr * sign[:, None]
    Q = torch.tensor([9.0, 9.0, -1.0], dtype=means.dtype, device=means.device)
    d = (Tw * Q * Tw).sum(1)
    d_safe = torch.where(d == 0, torch.ones_like(d), d)
    mx = (Tu * Q * Tw).sum(1) / d_safe
    my = (Tv * Q * Tw).sum(1) / d_safe
    with torch.no_grad():
        ex = torch.sqrt(torch.clamp(mx * mx - (Tu * Q * Tu).sum(1) / d_safe, min=1e-4))
        ey = torch.sqrt(torch.clamp(my * my - (Tv * Q * Tv).sum(1) / d_safe, min=1e-4))
        half = torch.maximum(torch.maximum(ex, ey), torch.full_like(ex, 3 * 0.707106))
        radius = torch.ceil(half)
        ok = (pv[:, 2] > NEAR) & (facing != 0) & (d != 0) & torch.isfinite(mx) & torch.isfinite(my) & (radius < 1e7)
        radius = torch.where(ok, radius, torch.zeros_like(radius))
        # the integer radius is ambiguous when the half extent sits within float32 rounding of an integer: half^2 is a
        # difference of terms of size mean2D^2 (~1e6 at 1080p), so its error scales with them
        big = mx * mx + my * my + ((Tu * Q * Tu).sum(1) / d_safe).abs() + ((Tv * Q * Tv).sum(1) / d_safe).abs()
        tol = 1e-6 * big / (2 * half) + 1e-5 * half
        frac = half - torch.floor(half)
        rad_amb = ok & (half > 3 * 0.707106 + 1e-6) & ((frac < tol) | (frac > 1 - tol))
    return dict(P=P, W=W, H=H, pv=pv, R=R, Tu=Tu, Tv=Tv, Tw=Tw, nv=nv, mx=mx, my=my, d=d, radius=radius, ok=ok,
                rad_amb=rad_amb, depth32=pv[:, 2].detach().float())


def tile_rect(mx, my, r, W, H):
    """The reference's getRect on 16x16 tiles (float arithmetic of the kernel, truncation toward zero)."""
    gx, gy = (W + 15) // 16, (H + 15) // 16
    tr = lambda v: torch.trunc(v)
    x0 = torch.clamp(tr((mx - r) / 16), 0, gx); y0 = torch.clamp(tr((my - r) / 16), 0, gy)
    x1 = torch.clamp(tr((mx + r + 15) / 16), 0, gx); y1 = torch.clamp(tr((my + r + 15) / 16), 0, gy)
    return torch.stack([x0, y0, x1, y1], 1).long()


def rects(g, radius=None):
    """Nominal rect of every Gaussian (zero for culled ones / empty rects) and the area."""
    r = g["radius"] if radius is None else radius
    rc = tile_rect(g["mx"].detach(), g["my"].detach(), r, g["W"], g["H"])
    area = (rc[:, 2] - rc[:, 0]) * (rc[:, 3] - rc[:, 1])
    live = g["ok"] & (area > 0)
    rc = torch.where(live[:, None], rc, torch.zeros_like(rc))
    return rc, live


def render(g, opac, rgb, bg, pix=None, eps_px=1e-3, trace=False):
    """Composite the pixels pix[N,2] (integer x, y; default: all) -> dict(image[3,N], maps[9,N], flag[N],
    contrib[N] (number of blended splats)).  opac [P], rgb [P,3], bg [3].  trace: also the blend weight and depth of
    every Gaussian in compositing order (weights[K,N], depths[K,N]; weight 0 where it did not blend)."""
    W, H = g["W"], g["H"]
    dev, dt = g["Tu"].device, g["Tu"].dtype
    if pix is None:
        ys, xs = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij")
        pix = torch.stack([xs.flatten(), ys.flatten()], 1)
    N = pix.shape[0]
    fx, fy = pix[:, 0].to(dt), pix[:, 1].to(dt)
    tx, ty = pix[:, 0] // 16, pix[:, 1] // 16
    rc, live = rects(g)
    # rect ambiguity: rects with the centre moved by eps_px (and the radius by one when it is ambiguous)
    with torch.no_grad():
        r0 = g["radius"]
        lo_r = torch.where(g["rad_amb"], r0 - 1, r0)
        hi_r = torch.where(g["rad_amb"], r0 + 1, r0)
        cands = [tile_rect(g["mx"].detach() + sx, g["my"].detach() + sy, rr, W, H)
                 for sx in (-eps_px, eps_px) for sy in (-eps_px, eps_px) for rr in (lo_r, hi_r)]
    # only Gaussians whose rect (or a plausible one) meets a tile of the requested pixels matter
    with torch.no_grad():
        keep = torch.zeros_like(live)
        for t in torch.unique(ty * 65536 + tx).tolist():
            a, b = t % 65536, t // 65536
            for c in cands + [rc]:
                keep |= (a >= c[:, 0]) & (a < c[:, 2]) & (b >= c[:, 1]) & (b < c[:, 3])
    idx = torch.nonzero(live & keep).flatten()
    keys = g["depth32"][idx].double().cpu().tolist()
    order = [i for _, i in sorted(zip(keys, idx.tolist()))]
    z0 = torch.zeros(N, dtype=dt, device=dev)
    T = torch.ones(N, dtype=dt, device=dev)
    C = [z0.clone() for _ in range(3)]
    Nn = [z0.clone() for _ in range(3)]
    D, M1, M2, dist, med_z, med_w, med_id = (z0.clone() for _ in range(7))
    done = torch.zeros(N, dtype=torch.bool, device=dev)
    flag = torch.zeros(N, dtype=torch.bool, device=dev)
    contrib = torch.zeros(N, dtype=torch.long, device=dev)
    tw, tz = [], []
    for i in order:
        inr = (tx >= rc[i, 0]) & (tx < rc[i, 2]) & (ty >= rc[i, 1]) & (ty < rc[i, 3])
        ins = [(tx >= c[i, 0]) & (tx < c[i, 2]) & (ty >= c[i, 1]) & (ty < c[i, 3]) for c in cands]
        amb_rect = torch.zeros_like(inr)
        for m in ins:
            amb_rect |= m != inr
        Tu, Tv, Tw = g["Tu"][i], g["Tv"][i], g["Tw"][i]
        k = fx[:, None] * Tw[None] - Tu[None]
        l = fy[:, None] * Tw[None] - Tv[None]
        p = torch.linalg.cross(k, l, dim=1)
        pz_ok = p[:, 2] != 0
        pz = torch.where(pz_ok, p[:, 2], torch.ones_like(p[:, 2]))
        sx, sy = p[:, 0] / pz, p[:, 1] / pz
        rho3 = sx * sx + sy * sy
        rho2 = 2 * ((g["mx"][i] - fx) ** 2 + (g["my"][i] - fy) ** 2)
        use3 = (rho3 <= rho2).detach()
        rho = torch.where(use3, rho3, rho2)
        z = torch.where(use3, sx * Tw[0] + sy * Tw[1] + Tw[2], Tw[2].expand(N))
        zok = pz_ok & (z >= NEAR).detach()
        oG = opac[i] * torch.exp(-0.5 * rho)
        alpha = torch.clamp(oG, max=0.99)
        aok = zok & (alpha >= 1.0 / 255).detach()
        cand = inr & ~done
        act = cand & aok
        test_T = T * (1 - alpha)
        term = act & (test_T < 1e-4).detach()
        blend = act & ~term
        with torch.no_grad():
            live_pair = cand & pz_ok & (opac[i] * torch.exp(-0.5 * torch.minimum(rho3, rho2)) > 0.5 / 255)
            zmag = (sx * Tw[0]).abs() + (sy * Tw[1]).abs() + Tw[2].abs()
            f = live_pair & ((z - NEAR).abs() < 1e-5 * zmag)
            f |= live_pair & ((rho3 - rho2).abs() < 1e-3 * (rho3 + rho2) + 1e-9)
            f |= cand & zok & ((alpha - 1.0 / 255).abs() < REL / 255)
            f |= act & ((test_T - 1e-4).abs() < REL * 1e-4)
            f |= blend & ((T - 0.5).abs() < REL * 0.5)
            f |= act & ((oG - 0.99).abs() < 1e-4)
            f |= ~done & amb_rect & zok & (oG >= 0.5 / 255)  # a rect edge in doubt where the splat is visible
            flag |= f
        w = alpha * T
        zs = torch.where(blend, z, torch.ones_like(z))
        m = FAR / (FAR - NEAR) * (1 - NEAR / zs)
        A = 1 - T
        for c in range(3):
            C[c] = torch.where(blend, C[c] + rgb[i, c] * w, C[c])
            Nn[c] = torch.where(blend, Nn[c] + g["nv"][i, c] * w, Nn[c])
        D = torch.where(blend, D + z * w, D)
        dist = torch.where(blend, dist + (m * m * A + M2 - 2 * m * M1) * w, dist)
        M1 = torch.where(blend, M1 + m * w, M1)
        M2 = torch.where(blend, M2 + m * m * w, M2)
        med = blend & (T > 0.5).detach()
        med_z = torch.where(med, z, med_z)
        med_w = torch.where(med, w, med_w)
        med_id = torch.where(med, torch.full_like(med_id, float(i)), med_id)
        T = torch.where(blend, test_T, T)
        contrib = contrib + blend.long()
        done = done | term
        if trace:
            tw.append(torch.where(blend, w, z0).detach()); tz.append(zs.detach())
    image = torch.stack([C[c] + T * bg[c] for c in range(3)])
    maps = torch.stack([D, 1 - T, Nn[0], Nn[1], Nn[2], med_z, dist, med_w, med_id])
    out = dict(image=image, maps=maps, flag=flag, contrib=contrib, pix=pix, order=order)
    if trace:
        out["weights"], out["depths"] = torch.stack(tw) if tw else z0[None], torch.stack(tz) if tz else z0[None] + 1
    return out


def scene_tensors(s, device, dtype=torch.float64):
    """Float64 copies of a surfel scene's inputs (tests/surfel_scenes.py)."""
    t = lambda k: torch.tensor(s[k], dtype=dtype, device=device)
    out = {k: t(k) for k in ("means3D", "scales", "rotations", "opacities", "viewmatrix", "projmatrix", "campos", "bg")}
    out["shs"] = t("shs") if "shs" in s else None
    out["colors_precomp"] = t("colors_precomp") if "colors_precomp" in s else None
    return out


def run(s, device="cpu", pix=None, grads=False, upstream=None, trace=False):
    """Forward (and optionally autograd backward) of a scene dict -> results.  upstream = (dL_dimage[3,N],
    dL_dmaps[7,N]) in the pixel order of `pix`; flagged pixels get zero upstream."""
    t = scene_tensors(s, device)
    leaves = {}
    if grads:
        for k in ("means3D", "scales", "rotations", "opacities", "shs", "colors_precomp"):
            if t[k] is not None:
                t[k].requires_grad_(True)
                leaves[k] = t[k]
        delta = torch.zeros(t["means3D"].shape[0], 2, dtype=torch.float64, device=device, requires_grad=True)
        leaves["delta"] = delta
    else:
        delta = None
    g = project(t["means3D"], t["scales"], t["rotations"], t["viewmatrix"], t["projmatrix"], s["W"], s["H"],
                s["scale_modifier"], delta)
    rgb = t["colors_precomp"] if t["colors_precomp"] is not None else sh_colors(t["shs"], s["D"], t["means3D"], t["campos"])
    out = render(g, t["opacities"].reshape(-1), rgb, t["bg"], pix, trace=trace)
    out["geom"] = g
    if grads:
        gi, gm = upstream
        keep = (~out["flag"]).to(gi.dtype)
        loss = (out["image"] * gi * keep).sum() + (out["maps"][:7] * gm * keep).sum()
        loss.backward()
        out["grads"] = {k: v.grad for k, v in leaves.items()}
        # means2D statistic in NDC units, as gsr_surfel_backward reports it
        dd = leaves["delta"].grad
        out["grads"]["means2D"] = torch.stack([dd[:, 0] * s["W"] / 2, dd[:, 1] * s["H"] / 2], 1)
    return out


def pairwise_distortion(w, m):
    """sum_{i<j} w_i w_j (m_i - m_j)^2 of one pixel's blend weights and normalised depths."""
    n = len(w)
    return sum(w[i] * w[j] * (m[i] - m[j]) ** 2 for i in range(n) for j in range(i + 1, n))


def m_of(z):
    return FAR / (FAR - NEAR) * (1 - NEAR / z)
