// Scaffold-GS neural-Gaussian decoding (the scaffold_renderer): what follows the anchor MLPs.  The reference turns the
// MLP outputs into Gaussians with ~25 torch launches (repeat, a [Nv*k, 22] concatenation, boolean-mask gathers, one
// host synchronisation per mask index); here it is a count + prefix (one host read of the total M), one decode kernel
// and one backward kernel.  Contract (include/gsr.h, DESIGN.md §7d): for visible anchor v = vis[i] and offset j, with
// o = opacity[i,j], c = color[i,3j..3j+2], s = cov[i,7j..7j+6], S = scaling[v] (6 activated scales):
//   kept iff o > 0; rows anchor-major, offset-minor (the reference's mask order)
//   xyz = anchor[v] + offset[v,j] * S[0:3]    scales = S[3:6] * sigmoid(s[0:3])
//   rot = s[3:7] / max(|s[3:7]|, 1e-12)        rgb = c, opacity = o
// Products and sums are rounded one at a time (no contraction), as the torch ops of the reference round them.
#include "../../include/gsr.h"
#include "gsr_internal.cuh"

namespace gsr {

namespace {

using cta::SCAN_THREADS;  // anchors per block of the count
using cta::cta_exclusive_scan;
constexpr int DEC_THREADS = 256;

struct ScaffoldDecodeArgs {
  int Nv, k;
  const long long* vis;
  const int* base;
  const float *anchor, *offset, *scaling, *opacity, *color, *cov;
  float *xyz, *rgb, *out_opacity, *scales, *rotations;
};
struct ScaffoldDecodeBwdArgs {
  int Nv, k;
  const long long* vis;
  const int* base;
  const float *offset, *scaling, *opacity, *cov;
  const float *dL_dxyz, *dL_drgb, *dL_dopacity, *dL_dscales, *dL_drotations;
  float *dL_dopacity_mlp, *dL_dcolor, *dL_dcov, *dL_danchor, *dL_doffset, *dL_dscaling;
};

// per anchor: survivors of its k offsets; CTA-local exclusive prefix into base[i], CTA total into block_sum
__global__ void __launch_bounds__(SCAN_THREADS) k_scaffold_count(int Nv, int k, const float* __restrict__ opacity,
                                                                 int* __restrict__ base, int* __restrict__ block_sum) {
  const int i = blockIdx.x * SCAN_THREADS + threadIdx.x;
  int n = 0;
  if (i < Nv)
    for (int j = 0; j < k; j++) n += opacity[(size_t)i * k + j] > 0.f;
  int total;
  const int ex = cta_exclusive_scan(n, &total);
  if (i < Nv) base[i] = ex;
  if (threadIdx.x == 0) block_sum[blockIdx.x] = total;
}

// one CTA: exclusive prefix of the block totals in place, and the grand total M into base[Nv]
__global__ void __launch_bounds__(SCAN_THREADS) k_scaffold_scan_blocks(int nb, int Nv, int* __restrict__ block_sum,
                                                                       int* __restrict__ base) {
  int carry = 0;
  for (int b0 = 0; b0 < nb; b0 += SCAN_THREADS) {
    const int b = b0 + threadIdx.x;
    const int v = b < nb ? block_sum[b] : 0;
    int total;
    const int ex = cta_exclusive_scan(v, &total);
    if (b < nb) block_sum[b] = carry + ex;
    carry += total;
  }
  if (threadIdx.x == 0) base[Nv] = carry;
}

__global__ void __launch_bounds__(SCAN_THREADS) k_scaffold_add_blocks(int Nv, const int* __restrict__ block_sum,
                                                                      int* __restrict__ base) {
  const int i = blockIdx.x * SCAN_THREADS + threadIdx.x;
  if (i < Nv) base[i] += block_sum[blockIdx.x];
}

// one thread per (visible anchor, offset) pair: consecutive lanes write consecutive rows
__global__ void __launch_bounds__(DEC_THREADS) k_scaffold_decode(ScaffoldDecodeArgs a) {
  const long long t = (long long)blockIdx.x * DEC_THREADS + threadIdx.x;
  if (t >= (long long)a.Nv * a.k) return;
  const int i = (int)(t / a.k), j = (int)(t - (long long)i * a.k);
  const float o = a.opacity[t];
  if (!(o > 0.f)) return;
  int row = a.base[i];
  for (int jj = 0; jj < j; jj++) row += a.opacity[t - j + jj] > 0.f;  // rank among the anchor's survivors (L1 hits)
  const long long v = a.vis[i];
  const float* S = a.scaling + v * 6;
  const float* off = a.offset + (v * a.k + j) * 3;
  const float* anc = a.anchor + v * 3;
#pragma unroll
  for (int c = 0; c < 3; c++) a.xyz[3 * (size_t)row + c] = __fadd_rn(anc[c], __fmul_rn(off[c], S[c]));
  const float* col = a.color + t * 3;
#pragma unroll
  for (int c = 0; c < 3; c++) a.rgb[3 * (size_t)row + c] = col[c];
  a.out_opacity[row] = o;
  const float* s = a.cov + t * 7;
#pragma unroll
  for (int c = 0; c < 3; c++) a.scales[3 * (size_t)row + c] = __fmul_rn(S[3 + c], sigmoid_rn(s[c]));
  const float q0 = s[3], q1 = s[4], q2 = s[5], q3 = s[6];
  const float n = fmaxf(sqrtf(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(q0, q0), __fmul_rn(q1, q1)), __fmul_rn(q2, q2)),
                                        __fmul_rn(q3, q3))), 1e-12f);
  reinterpret_cast<float4*>(a.rotations)[row] =
      make_float4(__fdiv_rn(q0, n), __fdiv_rn(q1, n), __fdiv_rn(q2, n), __fdiv_rn(q3, n));
}

// one thread per visible anchor, its k offsets in order: the per-anchor sums need no atomics and are deterministic
__global__ void __launch_bounds__(DEC_THREADS) k_scaffold_decode_bwd(ScaffoldDecodeBwdArgs a) {
  const int i = blockIdx.x * DEC_THREADS + threadIdx.x;
  if (i >= a.Nv) return;
  const long long v = a.vis[i];
  const float* S = a.scaling + v * 6;
  float dA[3] = {0.f, 0.f, 0.f}, dS[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  int row = a.base[i];
  for (int j = 0; j < a.k; j++) {
    const long long t = (long long)i * a.k + j;
    float* d_s = a.dL_dcov + t * 7;
    float* d_c = a.dL_dcolor + t * 3;
    float* d_off = a.dL_doffset + (v * a.k + j) * 3;
    if (!(a.opacity[t] > 0.f)) {  // dropped: no path to any input
      a.dL_dopacity_mlp[t] = 0.f;
#pragma unroll
      for (int c = 0; c < 3; c++) d_c[c] = 0.f;
#pragma unroll
      for (int c = 0; c < 7; c++) d_s[c] = 0.f;
      continue;  // d_off stays as zeroed by the entry point
    }
    a.dL_dopacity_mlp[t] = a.dL_dopacity[row];
#pragma unroll
    for (int c = 0; c < 3; c++) d_c[c] = a.dL_drgb[3 * (size_t)row + c];
    const float* off = a.offset + (v * a.k + j) * 3;
#pragma unroll
    for (int c = 0; c < 3; c++) {  // xyz = anchor + offset * S[0:3]
      const float g = a.dL_dxyz[3 * (size_t)row + c];
      dA[c] += g;
      dS[c] += g * off[c];
      d_off[c] = g * S[c];
    }
    const float* s = a.cov + t * 7;
#pragma unroll
    for (int c = 0; c < 3; c++) {  // scales = S[3:6] * sigmoid(s[0:3])
      const float g = a.dL_dscales[3 * (size_t)row + c];
      const float sg = sigmoid_rn(s[c]);
      dS[3 + c] += g * sg;
      d_s[c] = g * S[3 + c] * sg * (1.f - sg);
    }
    // rot = q / max(|q|, 1e-12): d/dq = (g - r (r.g)) / |q|, or g / 1e-12 where the clamp holds the norm constant
    const float q[4] = {s[3], s[4], s[5], s[6]};
    const float nq = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    const float n = fmaxf(nq, 1e-12f), inv = 1.f / n;
    float g[4], r[4], dot = 0.f;
#pragma unroll
    for (int c = 0; c < 4; c++) {
      g[c] = a.dL_drotations[4 * (size_t)row + c];
      r[c] = q[c] * inv;
      dot += r[c] * g[c];
    }
    const bool clamped = !(nq > 1e-12f);
#pragma unroll
    for (int c = 0; c < 4; c++) d_s[3 + c] = clamped ? g[c] * inv : (g[c] - r[c] * dot) * inv;
    row++;
  }
#pragma unroll
  for (int c = 0; c < 3; c++) a.dL_danchor[v * 3 + c] = dA[c];
#pragma unroll
  for (int c = 0; c < 6; c++) a.dL_dscaling[v * 6 + c] = dS[c];
}

}  // namespace

}  // namespace gsr

using namespace gsr;

namespace {
bool scaffold_k_ok(int k) { return k >= 1 && k <= 32; }
}  // namespace

extern "C" {

int gsr_scaffold_visible(int N, const float* means3D, const float* scales, const float* rotations,
                         const float* cov3D_precomp, float scale_modifier, const float* viewmatrix,
                         const float* projmatrix, int width, int height, float tan_fovx, float tan_fovy,
                         float kernel_size, int* radii, void* stream) {
  const char* fn = "gsr_scaffold_visible";
  if (N < 0 || width <= 0 || height <= 0) return fail(fn, "N >= 0, width and height > 0");
  if (!kernel_size_ok(kernel_size)) return fail(fn, "kernel_size must be finite and >= 0");
  if (!means3D || !viewmatrix || !projmatrix || !radii || (!cov3D_precomp && (!scales || !rotations)))
    return fail(fn, "need means3D, the camera, radii and scales+rotations or cov3D_precomp");
  if (!cov3D_precomp && misaligned16(rotations)) return fail(fn, "rotations must be 16-byte aligned");
  if ((width + TILE_X - 1) / TILE_X > 65535 || (height + TILE_Y - 1) / TILE_Y > 65535) return fail(fn, "image too large");
  if (N == 0) return 0;
  ScaffoldVisArgs a{};
  a.P = N; a.W = width; a.H = height; a.means3D = means3D; a.cov3D_precomp = cov3D_precomp;
  a.scales = cov3D_precomp ? nullptr : scales; a.rotations = cov3D_precomp ? nullptr : rotations;
  a.view = viewmatrix; a.proj = projmatrix; a.scale_modifier = scale_modifier; a.tan_fovx = tan_fovx;
  a.tan_fovy = tan_fovy; a.kernel_size = kernel_size; a.radii = radii;
  launch_scaffold_visible(a, (cudaStream_t)stream);
  return launched(fn);
}

int gsr_scaffold_count(int Nv, int k, const float* opacity, int* base, int* scratch, void* stream) {
  const char* fn = "gsr_scaffold_count";
  if (Nv < 0 || !scaffold_k_ok(k)) return fail(fn, "Nv >= 0 and 1 <= k <= 32");
  if ((long long)Nv * k > 0x7fffffffll) return fail(fn, "Nv * k must fit in int32");
  if (!base || (Nv > 0 && (!opacity || !scratch))) return fail(fn, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (Nv == 0) return check(cudaMemsetAsync(base, 0, sizeof(int), st), fn) ? 0 : -1;
  const int nb = (Nv + SCAN_THREADS - 1) / SCAN_THREADS;
  k_scaffold_count<<<nb, SCAN_THREADS, 0, st>>>(Nv, k, opacity, base, scratch);
  k_scaffold_scan_blocks<<<1, SCAN_THREADS, 0, st>>>(nb, Nv, scratch, base);
  k_scaffold_add_blocks<<<nb, SCAN_THREADS, 0, st>>>(Nv, scratch, base);
  return launched(fn);
}

int gsr_scaffold_decode(int Nv, int k, const int64_t* vis, const int* base, const float* anchor, const float* offset,
                        const float* scaling, const float* opacity, const float* color, const float* cov, float* xyz,
                        float* rgb, float* out_opacity, float* scales, float* rotations, void* stream) {
  const char* fn = "gsr_scaffold_decode";
  if (Nv < 0 || !scaffold_k_ok(k)) return fail(fn, "Nv >= 0 and 1 <= k <= 32");
  if ((long long)Nv * k > 0x7fffffffll) return fail(fn, "Nv * k must fit in int32");
  if (Nv == 0) return 0;
  if (!vis || !base || !anchor || !offset || !scaling || !opacity || !color || !cov) return fail(fn, "null pointer");
  if (misaligned16(rotations)) return fail(fn, "rotations must be 16-byte aligned");
  ScaffoldDecodeArgs a{};
  a.Nv = Nv; a.k = k; a.vis = reinterpret_cast<const long long*>(vis); a.base = base; a.anchor = anchor;
  a.offset = offset; a.scaling = scaling; a.opacity = opacity; a.color = color; a.cov = cov; a.xyz = xyz; a.rgb = rgb;
  a.out_opacity = out_opacity; a.scales = scales; a.rotations = rotations;
  const long long n = (long long)Nv * k;
  k_scaffold_decode<<<blocks(n, DEC_THREADS), DEC_THREADS, 0, (cudaStream_t)stream>>>(a);
  return launched(fn);
}

int gsr_scaffold_decode_backward(int N, int Nv, int k, const int64_t* vis, const int* base, const float* offset,
                                 const float* scaling, const float* opacity, const float* cov, const float* dL_dxyz,
                                 const float* dL_drgb, const float* dL_dopacity, const float* dL_dscales,
                                 const float* dL_drotations, float* dL_dopacity_mlp, float* dL_dcolor, float* dL_dcov,
                                 float* dL_danchor, float* dL_doffset, float* dL_dscaling, void* stream) {
  const char* fn = "gsr_scaffold_decode_backward";
  if (N < 0 || Nv < 0 || Nv > N || !scaffold_k_ok(k)) return fail(fn, "0 <= Nv <= N and 1 <= k <= 32");
  if ((long long)N * k > 0x7fffffffll) return fail(fn, "N * k must fit in int32");
  if (N > 0 && (!dL_danchor || !dL_doffset || !dL_dscaling)) return fail(fn, "null pointer");
  if (Nv > 0 && (!vis || !base || !offset || !scaling || !opacity || !cov || !dL_dopacity_mlp || !dL_dcolor ||
                 !dL_dcov))
    return fail(fn, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (N == 0) return 0;
  // anchors that are not visible, and dropped offsets of visible ones, get exact zeros
  if (!check(cudaMemsetAsync(dL_danchor, 0, sizeof(float) * 3 * (size_t)N, st), fn) ||
      !check(cudaMemsetAsync(dL_doffset, 0, sizeof(float) * 3 * (size_t)N * k, st), fn) ||
      !check(cudaMemsetAsync(dL_dscaling, 0, sizeof(float) * 6 * (size_t)N, st), fn))
    return -1;
  if (Nv == 0) return 0;
  ScaffoldDecodeBwdArgs a{};
  a.Nv = Nv; a.k = k; a.vis = reinterpret_cast<const long long*>(vis); a.base = base; a.offset = offset;
  a.scaling = scaling; a.opacity = opacity; a.cov = cov; a.dL_dxyz = dL_dxyz; a.dL_drgb = dL_drgb;
  a.dL_dopacity = dL_dopacity; a.dL_dscales = dL_dscales; a.dL_drotations = dL_drotations;
  a.dL_dopacity_mlp = dL_dopacity_mlp; a.dL_dcolor = dL_dcolor; a.dL_dcov = dL_dcov; a.dL_danchor = dL_danchor;
  a.dL_doffset = dL_doffset; a.dL_dscaling = dL_dscaling;
  k_scaffold_decode_bwd<<<blocks(Nv, DEC_THREADS), DEC_THREADS, 0, st>>>(a);
  return launched(fn);
}

}  // extern "C"
