"""Float64 restatement of the contribution statistics of gsr_contribution, on the per-pixel walk of comp_ref64.

For one view and every Gaussian i, over the pixels of its tiles (comp_ref64.Compositing: the same tile lists, thresholds
and walk):
  weight[i] = sum of w = alpha T over the pixels where i blended,
  count[i]  = pixels where i blended + pixels that i ended (the first pair whose T (1 - alpha) < 1e-4; it does not blend),
  max[i]    = largest such w.

Error bound (DESIGN.md §7l).  With u = 2^-24 and, per blended pair, comp_ref64's gain g + K (g = 1 + M the pair's
conic-form magnitude, K the pixel's transmittance error gain):
  * alpha is within 5 u g of float64 and the forward's T within 5 u K, so w = fl(alpha T) is within 6 u (g + K) w;
    EPS_W = 1e-6 (~17 u) covers it with the second-order terms;
  * each w is rounded once to 32.32 fixed point (<= 2^-33); the integer sums are exact;
  * the per-view sum is converted to double and added to the total: 2^-52 relative per view.
So |weight - weight64| <= sum over pairs of (EPS_W (g + K) w + 2^-33) + views 2^-52 weight64 (`bound`), and
|max - max64| <= the largest EPS_W (g + K) w of the Gaussian (`max_bound`); count is exact.

Ambiguity.  At a pixel comp_ref64 flags (alpha vs 1/255, power vs 0, T (1 - alpha) vs 1e-4 within float32 rounding),
float32 may take the other decision and every later decision of the pixel can move.  Every Gaussian that could reach
the transmittance test at a flagged pixel (power <= FLAG_TOL M and o G >= (1 - FLAG_TOL g) / 255) is `tainted`; the
comparison skips tainted Gaussians and is exact-or-bounded for all others.
"""
import torch

import comp_ref64 as R

F64 = torch.float64
EPS_W = 1e-6
FIX_HALF_ULP = 2.0 ** -33


class Statistics:
    """Accumulates views: add(comp) for each comp_ref64.Compositing of a view."""

    def __init__(self, P):
        self.P = P
        self.views = 0
        self.weight = torch.zeros(P, dtype=F64)
        self.count = torch.zeros(P, dtype=torch.int64)
        self.max = torch.zeros(P, dtype=F64)
        self.bound = torch.zeros(P, dtype=F64)
        self.max_bound = torch.zeros(P, dtype=F64)
        self.tainted = torch.zeros(P, dtype=torch.bool)

    def add(self, comp):
        assert comp.P == self.P
        self.views += 1
        for tl in comp.tiles:
            ids, pid, ct, w, gain, stop = tl["ids"], tl["pid"], tl["contrib"], tl["w"], tl["gain"], tl["stop_pos"]
            n = ids.numel()
            w = torch.where(ct, w, torch.zeros_like(w))
            self.weight.index_add_(0, ids, w.sum(0))
            self.count.index_add_(0, ids, ct.sum(0))
            ended = stop < n
            if ended.any():
                self.count.index_add_(0, ids[stop[ended]], torch.ones(int(ended.sum()), dtype=torch.int64))
            self.max.scatter_reduce_(0, ids, w.max(0).values, "amax")
            ew = EPS_W * gain * w
            self.bound.index_add_(0, ids, (ew + FIX_HALF_ULP * ct).sum(0))
            self.max_bound.scatter_reduce_(0, ids, ew.max(0).values, "amax")
            fl = comp.flag[pid]
            if fl.any():
                dx, dy = tl["dx"][fl], tl["dy"][fl]
                A, B, C, o = (comp.co[ids, j][None, :] for j in range(4))
                power = -0.5 * (A * dx * dx + C * dy * dy) - B * dx * dy
                M = 0.5 * A.abs() * dx * dx + 0.5 * C.abs() * dy * dy + (B * dx * dy).abs()
                oG = o * torch.exp(torch.clamp(power, max=0.0))
                cand = (power <= R.FLAG_TOL * M) & (oG >= R.ALPHA_MIN * (1 - R.FLAG_TOL * (1 + M)))
                self.tainted[ids[cand.any(0)]] = True
        return self

    def weight_bound(self):
        return self.bound + self.views * 2.0 ** -52 * self.weight


def brute_force(means2D, conic_opacity, depths, radii, W, H):
    """The same statistics from a scalar loop over every pixel and its tile's list (tests of this module only)."""
    import numpy as np
    m2 = np.asarray(means2D, np.float64).reshape(-1, 2)
    co = np.asarray(conic_opacity, np.float64).reshape(-1, 4)
    P = m2.shape[0]
    lists, gx, _ = R.tile_lists(means2D, radii, depths, W, H)
    weight, count, mx = np.zeros(P), np.zeros(P, np.int64), np.zeros(P)
    for y in range(H):
        for x in range(W):
            T = 1.0
            for i in lists[(y // R.TILE) * gx + x // R.TILE]:
                dx, dy = m2[i, 0] - x, m2[i, 1] - y
                A, B, C, o = co[i]
                power = -0.5 * (A * dx * dx + C * dy * dy) - B * dx * dy
                if power > 0:
                    continue
                alpha = min(R.ALPHA_MAX, o * np.exp(power))
                if alpha < R.ALPHA_MIN:
                    continue
                count[i] += 1
                if T * (1 - alpha) < R.T_MIN:
                    break
                weight[i] += alpha * T
                mx[i] = max(mx[i], alpha * T)
                T *= 1 - alpha
    return weight, count, mx
