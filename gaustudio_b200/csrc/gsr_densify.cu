// Adaptive density control of 3DGS / 2DGS training (graphdeco's densify_and_prune, DESIGN.md §7e): the screen-space
// statistics of every view, and the clone / split / prune of a densification step as one count + prefix (one host read
// of four totals) and one launch that writes every output tensor.
//   grad = accum / denom (NaN -> 0)     smax = max_c exp(scale[c])     t_clone = percent_dense * extent
//   clone iff grad >= max_grad and smax <= t_clone     split iff grad >= max_grad and smax > t_clone
//   child scale = log(exp(scale) * (1 / 1.6f))    child xyz = R(rot) (z (.) exp(scale)) + xyz
//   prune iff sigmoid(opacity) < min_opacity, or (prune_big) smax > t_big, on the row's own values
// Row order: surviving originals, surviving clones (source order), first children, second children (split order).
// Every decision and every value except the children's xyz is rounded op by op as torch's CUDA kernels round them.
#include "../../include/gsr.h"
#include "gsr_internal.cuh"

#include <cmath>

namespace gsr {

namespace {

using cta::SCAN_THREADS;  // Gaussians per block of the count
using cta::cta_exclusive_scan;
constexpr int STATS_THREADS = 256;
constexpr int APPLY_THREADS = 256;
constexpr int APPLY_ITEMS = 4;  // elements per thread of the apply kernel
constexpr int NCAT = 4;         // per-Gaussian counts: original kept, clone kept, child pair kept, split
constexpr int F_ORIG = 1, F_CLONE = 2, F_PAIR = 4, F_SPLIT = 8;
// torch divides a CUDA tensor by a Python scalar as a product with the scalar's float reciprocal
constexpr float kInvSplit = 1.0f / 1.6f;

// scratch (int32): totals[4] | prefix[4][P] | flags[P] | block sums[4][nb]
struct ScratchView {
  int* totals;
  int* pre;
  int* flags;
  int* bsum;
};
__host__ __device__ inline ScratchView carve_scratch(int* s, int P, int nb) {
  return {s, s + NCAT, s + NCAT + (size_t)NCAT * P, s + NCAT + (size_t)(NCAT + 1) * P};
}

// NaN-propagating max, like torch.max
__device__ __forceinline__ float max_nan(float a, float b) { return (b > a || b != b) ? b : a; }

__device__ __forceinline__ float child_log_scale(float s) { return logf(__fmul_rn(expf(s), kInvSplit)); }

__global__ void __launch_bounds__(STATS_THREADS) k_densify_stats(int P, const float* __restrict__ grad,
                                                                const int* __restrict__ radii, float* __restrict__ accum,
                                                                float* __restrict__ denom, float* __restrict__ max_r) {
  const int i = blockIdx.x * STATS_THREADS + threadIdx.x;
  if (i >= P) return;
  const int r = radii[i];
  if (!(r > 0)) return;
  const float gx = grad[3 * (size_t)i], gy = grad[3 * (size_t)i + 1];
  accum[i] = __fadd_rn(accum[i], sqrtf(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy))));
  denom[i] = __fadd_rn(denom[i], 1.f);
  const float m = max_r[i];
  max_r[i] = max_nan(m, (float)r);
}

struct CountArgs {
  int P, sd, prune_big;
  const float *accum, *denom, *scale, *opacity;
  float max_grad, min_opacity, t_clone, t_big;
};

// per Gaussian: its flags and the four counts; CTA-local exclusive prefixes, CTA totals into the block sums
__global__ void __launch_bounds__(SCAN_THREADS) k_densify_count(CountArgs a, ScratchView s, int nb) {
  const int i = blockIdx.x * SCAN_THREADS + threadIdx.x;
  int f = 0;
  if (i < a.P) {
    float g = __fdiv_rn(a.accum[i], a.denom[i]);
    if (g != g) g = 0.f;
    float smax = -INFINITY, cmax = -INFINITY;
    for (int c = 0; c < a.sd; c++) {
      const float sc = a.scale[(size_t)i * a.sd + c];
      smax = max_nan(smax, expf(sc));
      cmax = max_nan(cmax, expf(child_log_scale(sc)));
    }
    const bool sel = g >= a.max_grad;
    const bool clone = sel && smax <= a.t_clone, split = sel && smax > a.t_clone;
    const bool faint = sigmoid_rn(a.opacity[i]) < a.min_opacity;
    const bool prune_self = faint || (a.prune_big && smax > a.t_big);
    const bool prune_child = faint || (a.prune_big && cmax > a.t_big);
    f = (!split && !prune_self ? F_ORIG : 0) | (clone && !prune_self ? F_CLONE : 0) |
        (split && !prune_child ? F_PAIR : 0) | (split ? F_SPLIT : 0);
    s.flags[i] = f;
  }
#pragma unroll
  for (int c = 0; c < NCAT; c++) {
    int total;
    const int ex = cta_exclusive_scan((f >> c) & 1, &total);
    if (i < a.P) s.pre[(size_t)c * a.P + i] = ex;
    if (threadIdx.x == 0) s.bsum[(size_t)c * nb + blockIdx.x] = total;
  }
}

// CTA c: exclusive prefix of category c's block totals in place, and its grand total
__global__ void __launch_bounds__(SCAN_THREADS) k_densify_scan_blocks(ScratchView s, int nb) {
  int* bs = s.bsum + (size_t)blockIdx.x * nb;
  int carry = 0;
  for (int b0 = 0; b0 < nb; b0 += SCAN_THREADS) {
    const int b = b0 + threadIdx.x;
    const int v = b < nb ? bs[b] : 0;
    int total;
    const int ex = cta_exclusive_scan(v, &total);
    if (b < nb) bs[b] = carry + ex;
    carry += total;
  }
  if (threadIdx.x == 0) s.totals[blockIdx.x] = carry;
}

__global__ void __launch_bounds__(SCAN_THREADS) k_densify_add_blocks(int P, ScratchView s, int nb) {
  const int i = blockIdx.x * SCAN_THREADS + threadIdx.x;
  if (i >= P) return;
#pragma unroll
  for (int c = 0; c < NCAT; c++) s.pre[(size_t)c * P + i] += s.bsum[(size_t)c * nb + blockIdx.x];
}

struct ApplyTable {
  const float* src[GSR_DENSIFY_MAX_ENTRIES];
  float* dst[GSR_DENSIFY_MAX_ENTRIES];
  int width[GSR_DENSIFY_MAX_ENTRIES];
  int role[GSR_DENSIFY_MAX_ENTRIES];
  int rows_per_block[GSR_DENSIFY_MAX_ENTRIES];
  unsigned first_block[GSR_DENSIFY_MAX_ENTRIES + 1];
  int n;
  int P, sd, n_orig, n_clone, n_pair, n_split;
  const float *rot, *scale, *noise;  // the parents' rotation and log-scale rows, z [2 n_split, 3]
  const int *pre, *flags;
};

// child j's xyz component c: R(rot) (z[j] (.) exp(scale)) + xyz; build_rotation normalises by the plain L2 norm
__device__ __forceinline__ float child_xyz(const ApplyTable& t, int i, int c, int j, float x) {
  const float4 q4 = reinterpret_cast<const float4*>(t.rot)[i];
  const float n = sqrtf(q4.x * q4.x + q4.y * q4.y + q4.z * q4.z + q4.w * q4.w);
  const float r = q4.x / n, qx = q4.y / n, qy = q4.z / n, qz = q4.w / n;
  float R0, R1, R2;
  if (c == 0) {
    R0 = 1.f - 2.f * (qy * qy + qz * qz); R1 = 2.f * (qx * qy - r * qz); R2 = 2.f * (qx * qz + r * qy);
  } else if (c == 1) {
    R0 = 2.f * (qx * qy + r * qz); R1 = 1.f - 2.f * (qx * qx + qz * qz); R2 = 2.f * (qy * qz - r * qx);
  } else {
    R0 = 2.f * (qx * qz - r * qy); R1 = 2.f * (qy * qz + r * qx); R2 = 1.f - 2.f * (qx * qx + qy * qy);
  }
  const float* z = t.noise + 3 * (size_t)j;
  const float* s = t.scale + (size_t)i * t.sd;
  const float v0 = z[0] * expf(s[0]), v1 = z[1] * expf(s[1]), v2 = t.sd == 3 ? z[2] * expf(s[2]) : z[2] * 0.f;
  return R0 * v0 + R1 * v1 + R2 * v2 + x;
}

// one block per run of rows of one entry; consecutive threads take consecutive elements of the run, so reads are
// coalesced for every width and writes are coalesced wherever consecutive rows land in consecutive output rows
__global__ void __launch_bounds__(APPLY_THREADS) k_densify_apply(const __grid_constant__ ApplyTable t) {
  int e = 0;
  while (e + 1 < t.n && blockIdx.x >= t.first_block[e + 1]) e++;
  const int w = t.width[e], role = t.role[e];
  const int row0 = (int)(blockIdx.x - t.first_block[e]) * t.rows_per_block[e];
  const int nrows = min(t.rows_per_block[e], t.P - row0);
  const float* src = t.src[e] + (size_t)row0 * w;
  float* dst = t.dst[e];
  const int n = nrows * w;
  const int* pre_o = t.pre;
  const int* pre_c = t.pre + t.P;
  const int* pre_k = t.pre + 2 * (size_t)t.P;
  const int* pre_s = t.pre + 3 * (size_t)t.P;
  // a run holds APPLY_ITEMS elements per thread, or one row wider than that: the stride covers the whole run
  for (int l = threadIdx.x; l < n; l += APPLY_THREADS) {
    const int ri = l / w, c = l - ri * w, i = row0 + ri;
    const int f = t.flags[i];
    if (!f) continue;
    const float v = src[l];
    if (f & F_ORIG) dst[(size_t)pre_o[i] * w + c] = v;
    if (f & F_CLONE) dst[((size_t)t.n_orig + pre_c[i]) * w + c] = role == GSR_DENSIFY_MOMENT ? 0.f : v;
    if (f & F_PAIR) {
      const size_t r0 = (size_t)t.n_orig + t.n_clone + pre_k[i], r1 = r0 + t.n_pair;
      float v0 = v, v1 = v;
      if (role == GSR_DENSIFY_MOMENT) {
        v0 = v1 = 0.f;
      } else if (role == GSR_DENSIFY_SCALE) {
        v0 = v1 = child_log_scale(v);
      } else if (role == GSR_DENSIFY_XYZ) {
        const int q = pre_s[i];
        v0 = child_xyz(t, i, c, q, v);
        v1 = child_xyz(t, i, c, t.n_split + q, v);
      }
      dst[r0 * w + c] = v0;
      dst[r1 * w + c] = v1;
    }
  }
}

}  // namespace

}  // namespace gsr

using namespace gsr;

extern "C" {

int gsr_densify_stats(int P, const float* viewspace_grad, const int* radii, float* accum, float* denom,
                      float* max_radii2D, void* stream) {
  if (P < 0) return fail("gsr_densify_stats", "P >= 0");
  if (P == 0) return 0;
  if (!viewspace_grad || !radii || !accum || !denom || !max_radii2D) return fail("gsr_densify_stats", "null pointer");
  k_densify_stats<<<blocks(P, STATS_THREADS), STATS_THREADS, 0, (cudaStream_t)stream>>>(
      P, viewspace_grad, radii, accum, denom, max_radii2D);
  return launched("gsr_densify_stats");
}

int gsr_densify_count(int P, int scale_dim, const float* accum, const float* denom, const float* scale,
                      const float* opacity, float max_grad, float min_opacity, float clone_max_scale, int prune_big,
                      float big_scale, int* scratch, void* stream) {
  const char* fn = "gsr_densify_count";
  if (P < 0) return fail(fn, "P >= 0");
  if (scale_dim != 2 && scale_dim != 3) return fail(fn, "scale_dim must be 2 or 3");
  if (!scratch || (P > 0 && (!accum || !denom || !scale || !opacity))) return fail(fn, "null pointer");
  if (!std::isfinite(max_grad) || !std::isfinite(min_opacity) || !std::isfinite(clone_max_scale) ||
      (prune_big && !std::isfinite(big_scale)))
    return fail(fn, "thresholds must be finite");
  cudaStream_t st = (cudaStream_t)stream;
  if (P == 0) return check(cudaMemsetAsync(scratch, 0, NCAT * sizeof(int), st), fn) ? 0 : -1;
  const int nb = (P + SCAN_THREADS - 1) / SCAN_THREADS;
  const ScratchView s = carve_scratch(scratch, P, nb);
  CountArgs a{};
  a.P = P; a.sd = scale_dim; a.prune_big = prune_big != 0; a.accum = accum; a.denom = denom; a.scale = scale;
  a.opacity = opacity; a.max_grad = max_grad; a.min_opacity = min_opacity; a.t_clone = clone_max_scale;
  a.t_big = big_scale;
  k_densify_count<<<nb, SCAN_THREADS, 0, st>>>(a, s, nb);
  k_densify_scan_blocks<<<NCAT, SCAN_THREADS, 0, st>>>(s, nb);
  k_densify_add_blocks<<<nb, SCAN_THREADS, 0, st>>>(P, s, nb);
  return launched(fn);
}

int gsr_densify_apply(int P, int scale_dim, const int* scratch, int n_orig, int n_clone, int n_pair, int n_split,
                      const float* noise, int n_entries, const gsr_densify_entry* entries, void* stream) {
  const char* fn = "gsr_densify_apply";
  if (P < 0 || n_orig < 0 || n_clone < 0 || n_pair < 0 || n_split < n_pair || n_orig > P || n_clone > P ||
      n_split > P || (long long)n_orig + n_clone + 2ll * n_pair > 0x7fffffffll)
    return fail(fn, "counts out of range (P_new = n_orig + n_clone + 2 n_pair must fit in int32)");
  if (scale_dim != 2 && scale_dim != 3) return fail(fn, "scale_dim must be 2 or 3");
  if (n_entries < 1 || n_entries > GSR_DENSIFY_MAX_ENTRIES || !entries) return fail(fn, "1..24 entries");
  ApplyTable t{};
  int n_xyz = 0, n_scale = 0, n_rot = 0;
  const bool any_out = (long long)n_orig + n_clone + n_pair > 0;
  unsigned nb = 0;
  for (int k = 0; k < n_entries; k++) {
    const gsr_densify_entry& q = entries[k];
    if (q.role < GSR_DENSIFY_COPY || q.role > GSR_DENSIFY_MOMENT || q.width < 1 || q.width > 4096 ||
        (q.role == GSR_DENSIFY_XYZ && q.width != 3) || (q.role == GSR_DENSIFY_SCALE && q.width != scale_dim) ||
        (q.role == GSR_DENSIFY_ROT && q.width != 4))
      return fail(fn, "bad entry (role, or width: xyz 3, scale scale_dim, rotation 4, others 1..4096)");
    if ((P > 0 && !q.src) || (any_out && !q.dst)) return fail(fn, "null pointer");
    n_xyz += q.role == GSR_DENSIFY_XYZ; n_scale += q.role == GSR_DENSIFY_SCALE; n_rot += q.role == GSR_DENSIFY_ROT;
    t.src[k] = q.src; t.dst[k] = q.dst; t.width[k] = q.width; t.role[k] = q.role;
    t.rows_per_block[k] = max(1, APPLY_THREADS * APPLY_ITEMS / q.width);
    t.first_block[k] = nb;
    nb += blocks(P, t.rows_per_block[k]);
    if (q.role == GSR_DENSIFY_SCALE) t.scale = q.src;
    if (q.role == GSR_DENSIFY_ROT) t.rot = q.src;
  }
  if (n_xyz != 1 || n_scale != 1 || n_rot != 1) return fail(fn, "need exactly one xyz, one scale and one rotation entry");
  if (P > 0 && (!scratch || (n_split > 0 && !noise))) return fail(fn, "null pointer");
  if (P > 0 && misaligned16(t.rot)) return fail(fn, "rotations must be 16-byte aligned");
  if (P == 0 || !any_out) return 0;
  t.first_block[n_entries] = nb;
  t.n = n_entries; t.P = P; t.sd = scale_dim; t.n_orig = n_orig; t.n_clone = n_clone; t.n_pair = n_pair;
  t.n_split = n_split; t.noise = noise;
  const ScratchView s = carve_scratch(const_cast<int*>(scratch), P, (P + SCAN_THREADS - 1) / SCAN_THREADS);
  t.pre = s.pre; t.flags = s.flags;
  k_densify_apply<<<nb, APPLY_THREADS, 0, (cudaStream_t)stream>>>(t);
  return launched(fn);
}

}  // extern "C"
