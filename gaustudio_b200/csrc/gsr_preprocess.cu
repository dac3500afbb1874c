// Per-Gaussian stages: projection (forward), fused cov2D/projection/SH/cov3D backward, frustum marking.
//
// Restates, with the reference's floating-point expression order (so that nvcc contracts the same FMAs
// and radii / tile rects / depth keys come out bit-identical):
//   forward : $RAST/cuda_rasterizer/forward.cu:20-71 (SH), 74-113 (cov2D), 118-152 (cov3D), 155-256 (K1)
//   backward: $RAST/cuda_rasterizer/backward.cu:144-274 (K6), 346-412 (K7), 20-139 (SH), 278-341 (cov3D)
//   helpers : $RAST/cuda_rasterizer/auxiliary.h:41-77,107-117,139-164
// Design differences (H100): one packed 48-B splat record per Gaussian instead of five SoA arrays; per-tile
// instance counts are accumulated here (no per-Gaussian prefix scan, no duplicateWithKeys offsets); K6 and
// K7 are one kernel and write every output element (no torch::zeros pre-pass, rasterize_points.cu:160-169).
#include "gsr_internal.cuh"

#include <cstdio>

namespace gsr {

namespace {

// SH basis constants (auxiliary.h:22-39)
__device__ const float kC0 = 0.28209479177387814f;
__device__ const float kC1 = 0.4886025119029199f;
__device__ const float kC2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                                 -1.0925484305920792f, 0.5462742152960396f};
__device__ const float kC3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                                 0.3731763325901154f,  -0.4570457994644658f, 1.445305721320277f,
                                 -0.5900435899266435f};

struct V3 { float x, y, z; };

// ---- TMA (cp.async.bulk) staging of a CTA's contiguous SH block: PRE_THREADS Gaussians x (M-1) x 12 B of f_rest and
// PRE_THREADS x 12 B of f_dc land in shared memory while the threads do the projection math; rows of 3 / 45 words have
// odd strides, so per-thread row reads are bank-conflict free.  The backward fetches only the rows of the Gaussians that
// have a gradient into the same layout (gather_live_rows), writes its SH gradients into the same rows and ships the
// block with one bulk store per tensor.
// CTA size of the projection kernels: 128 measured best of 64 / 128 / 256 with several views in flight (A/B not
// repeated on the H100): smaller CTAs slot into the SMs as the compositing CTAs of other streams retire
#ifndef GSR_PRE_THREADS
#define GSR_PRE_THREADS 128
#endif
constexpr int PRE_THREADS = GSR_PRE_THREADS;
constexpr int SH_ROW = 52;  // floats per staged row of the un-fused [P,16,3] tensor: 192 B of data + 16 B pad (16-B aligned rows)
__device__ __forceinline__ unsigned smem_addr(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void bulk_load(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_addr(dst)), "l"(src), "r"(bytes), "r"(smem_addr(bar)) : "memory");
}
__device__ __forceinline__ void bulk_store(void* dst_gmem, const void* src_smem, unsigned bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem), "r"(smem_addr(src_smem)),
               "r"(bytes) : "memory");
}
__device__ __forceinline__ void bar_init_expect(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_addr(bar)) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
}
// every thread of the CTA stages its own row: barrier expects PRE_THREADS arrivals, each announcing its bytes
__device__ __forceinline__ void row_load(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
  bulk_load(dst, src, bytes, bar);
}
// a thread that stages nothing still arrives, announcing no bytes
__device__ __forceinline__ void bar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_addr(bar)) : "memory");
}
// Warp-cooperative gather of the warp's 32 consecutive rows of `row_bytes` (16-B aligned block, row_bytes >= 12) into
// the same layout in shared memory, in 16-B LDGSTS chunks: a chunk is fetched only if a row of `live` overlaps it (a
// chunk touches at most two rows).  Completes with cp.async.wait_all + __syncwarp.
__device__ __forceinline__ void gather_live_rows(float* dst, const float* src, unsigned row_bytes, unsigned live) {
  for (unsigned c = threadIdx.x & 31; c < 2 * row_bytes; c += 32) {  // 32 rows = 2 * row_bytes chunks
    const unsigned b = 16 * c, r = b / row_bytes;
    const unsigned rows = b + 16 > (r + 1) * row_bytes ? 3u : 1u;  // rows r and r + 1, or r alone
    if ((live >> r) & rows)
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_addr(dst + 4 * c)), "l"(src + 4 * c) : "memory");
  }
}
__device__ __forceinline__ void bar_wait0(unsigned long long* bar) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "PWAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], 0;\n"
      "@p bra PDONE;\n"
      "bra PWAIT;\n"
      "PDONE:\n"
      "}\n" ::"r"(smem_addr(bar)) : "memory");
}

// column-major 3x3, m[c][r]; product written in the accumulation order of glm's mat3*mat3
// (third_party/glm/glm/detail/type_mat3x3.inl:486-518) which the reference kernels inherit.
struct Mat3 { float m[3][3]; };
__device__ __forceinline__ Mat3 mmul(const Mat3& A, const Mat3& B) {
  Mat3 R;
#pragma unroll
  for (int c = 0; c < 3; c++)
#pragma unroll
    for (int r = 0; r < 3; r++)
      R.m[c][r] = A.m[0][r] * B.m[c][0] + A.m[1][r] * B.m[c][1] + A.m[2][r] * B.m[c][2];
  return R;
}
__device__ __forceinline__ Mat3 mtr(const Mat3& A) {
  Mat3 R;
#pragma unroll
  for (int c = 0; c < 3; c++)
#pragma unroll
    for (int r = 0; r < 3; r++) R.m[c][r] = A.m[r][c];
  return R;
}

__device__ __forceinline__ V3 xf4x3(const V3& p, const float* __restrict__ m) {
  V3 t;
  t.x = m[0] * p.x + m[4] * p.y + m[8] * p.z + m[12];
  t.y = m[1] * p.x + m[5] * p.y + m[9] * p.z + m[13];
  t.z = m[2] * p.x + m[6] * p.y + m[10] * p.z + m[14];
  return t;
}
__device__ __forceinline__ float4 xf4x4(const V3& p, const float* __restrict__ m) {
  float4 t;
  t.x = m[0] * p.x + m[4] * p.y + m[8] * p.z + m[12];
  t.y = m[1] * p.x + m[5] * p.y + m[9] * p.z + m[13];
  t.z = m[2] * p.x + m[6] * p.y + m[10] * p.z + m[14];
  t.w = m[3] * p.x + m[7] * p.y + m[11] * p.z + m[15];
  return t;
}

// auxiliary.h:41-44: the 1.0 / 0.5 literals make this a double-precision expression
__device__ __forceinline__ float ndc2pix(float v, int S) { return ((v + 1.0) * S - 1.0) * 0.5; }

// auxiliary.h:46-56
__device__ __forceinline__ void tile_rect(float px, float py, int max_radius, int gx, int gy, int& x0, int& y0,
                                          int& x1, int& y1) {
  x0 = min(gx, max((int)0, (int)((px - max_radius) / TILE_X)));
  y0 = min(gy, max((int)0, (int)((py - max_radius) / TILE_Y)));
  x1 = min(gx, max((int)0, (int)((px + max_radius + TILE_X - 1) / TILE_X)));
  y1 = min(gy, max((int)0, (int)((py + max_radius + TILE_Y - 1) / TILE_Y)));
}

struct Rot { Mat3 R; };
// rotation from the un-normalised quaternion (r,x,y,z) exactly as forward.cu:127-139 (quirk 2)
__device__ __forceinline__ Mat3 quat_mat(float r, float x, float y, float z) {
  Mat3 R;
  R.m[0][0] = 1.f - 2.f * (y * y + z * z);
  R.m[0][1] = 2.f * (x * y - r * z);
  R.m[0][2] = 2.f * (x * z + r * y);
  R.m[1][0] = 2.f * (x * y + r * z);
  R.m[1][1] = 1.f - 2.f * (x * x + z * z);
  R.m[1][2] = 2.f * (y * z - r * x);
  R.m[2][0] = 2.f * (x * z - r * y);
  R.m[2][1] = 2.f * (y * z + r * x);
  R.m[2][2] = 1.f - 2.f * (x * x + y * y);
  return R;
}
__device__ __forceinline__ Mat3 scale_mat(float sx, float sy, float sz) {
  Mat3 S;
#pragma unroll
  for (int c = 0; c < 3; c++)
#pragma unroll
    for (int r = 0; r < 3; r++) S.m[c][r] = 0.0f;
  S.m[0][0] = sx; S.m[1][1] = sy; S.m[2][2] = sz;
  return S;
}

// forward.cu:74-113 / backward.cu:160-197: everything the two call sites share
struct Cov2D {
  V3 t;
  float txtz, tytz, limx, limy;
  Mat3 T, Vrk, Wm, cov;
};
__device__ __forceinline__ void cov2d(const V3& mean, float fx, float fy, float tan_fovx, float tan_fovy,
                                      const float* cov3D, const float* __restrict__ view, Cov2D& o) {
  o.t = xf4x3(mean, view);
  o.limx = 1.3f * tan_fovx;
  o.limy = 1.3f * tan_fovy;
  o.txtz = o.t.x / o.t.z;
  o.tytz = o.t.y / o.t.z;
  o.t.x = min(o.limx, max(-o.limx, o.txtz)) * o.t.z;
  o.t.y = min(o.limy, max(-o.limy, o.tytz)) * o.t.z;
  Mat3 J;
  J.m[0][0] = fx / o.t.z; J.m[0][1] = 0.0f; J.m[0][2] = -(fx * o.t.x) / (o.t.z * o.t.z);
  J.m[1][0] = 0.0f; J.m[1][1] = fy / o.t.z; J.m[1][2] = -(fy * o.t.y) / (o.t.z * o.t.z);
  J.m[2][0] = 0; J.m[2][1] = 0; J.m[2][2] = 0;
  o.Wm.m[0][0] = view[0]; o.Wm.m[0][1] = view[4]; o.Wm.m[0][2] = view[8];
  o.Wm.m[1][0] = view[1]; o.Wm.m[1][1] = view[5]; o.Wm.m[1][2] = view[9];
  o.Wm.m[2][0] = view[2]; o.Wm.m[2][1] = view[6]; o.Wm.m[2][2] = view[10];
  o.T = mmul(o.Wm, J);
  o.Vrk.m[0][0] = cov3D[0]; o.Vrk.m[0][1] = cov3D[1]; o.Vrk.m[0][2] = cov3D[2];
  o.Vrk.m[1][0] = cov3D[1]; o.Vrk.m[1][1] = cov3D[3]; o.Vrk.m[1][2] = cov3D[4];
  o.Vrk.m[2][0] = cov3D[2]; o.Vrk.m[2][1] = cov3D[4]; o.Vrk.m[2][2] = cov3D[5];
  o.cov = mmul(mmul(mtr(o.T), mtr(o.Vrk)), o.T);
  o.cov.m[0][0] += 0.3f;
  o.cov.m[1][1] += 0.3f;
}

// Count helper: visits the binned tiles of every lane's rect.  Lanes with small rects (<= 32 tiles) loop themselves over
// the set bits of their tile mask; large rects (a splat covering much of the screen) are walked in full by the
// whole warp so one thread never serialises thousands of atomics (the reference's duplicateWithKeys does,
// rasterizer_impl.cu:98-108).
constexpr int kBigRect = 32;
template <typename F>
__device__ __forceinline__ void for_each_tile(int x0, int y0, int x1, int y1, uint32_t mask, int gx, F f) {
  const int w = x1 - x0, n = w * (y1 - y0);
  const unsigned lane = threadIdx.x & 31;
  if (n > 0 && n <= kBigRect) {
    while (mask) {
      const int i = __ffs(mask) - 1;
      mask &= mask - 1;
      f((y0 + i / w) * gx + x0 + i % w, lane);
    }
  }
  unsigned big = __ballot_sync(0xffffffffu, n > kBigRect);
  while (big) {
    const int src = __ffs(big) - 1;
    big &= big - 1;
    const int bx0 = __shfl_sync(0xffffffffu, x0, src), by0 = __shfl_sync(0xffffffffu, y0, src);
    const int bw = __shfl_sync(0xffffffffu, w, src), bn = __shfl_sync(0xffffffffu, n, src);
    for (int i = lane; i < bn; i += 32) f((by0 + i / bw) * gx + bx0 + i % bw, (unsigned)src);
  }
}

// Which tiles of a Gaussian's rect [x0,x1) x [y0,y1) (<= 32 tiles) can it contribute to at all?  Bit i (row-major in the
// rect) is set iff some point of tile i's pixel box lies in the ellipse E = {q(d) <= tau'}, q(d) = A dx^2 + 2B dx dy + C dy^2,
// d = pixel - mean, tau' = tau + margin (tau = 2 ln(255 o): alpha >= 1/255 needs q <= tau; the margin is the one of
// may_touch, taken over the whole rect).  Row by row instead of tile by tile: within the band dy in [lo, hi] of a tile
// row the ellipse spans dx in [xmin, xmax]; xmax(dy) = -(B/A) dy + sqrt((tau' - D dy^2) / A), D = C - B^2/A, is concave
// with its maximum hx = sqrt(tau' C / det) at dy = -B hx / C (and xmin mirrors it), so both follow from one clamped
// evaluation each, and the row's tiles are the contiguous run that overlaps [xmin, xmax] (convexity).  A superset of the
// contributing tiles is always safe: the compositing kernels apply the reference's per-pixel test.
__device__ __forceinline__ uint32_t tile_mask_of(float px, float py, float A, float B, float C, float opac, float tau,
                                                 int x0, int y0, int x1, int y1, int W, int H) {
  const int rw = x1 - x0;
  const uint32_t all = (rw * (y1 - y0) >= 32) ? 0xffffffffu : ((1u << (rw * (y1 - y0))) - 1u);
  if (opac < 0.0039f) return 0u;  // alpha <= o < 1/255 everywhere
  const float det = A * C - B * B;
  if (!(A > 1e-30f && C > 1e-30f && det > 0.f && A < 1e30f && C < 1e30f && tau >= 0.f)) return all;  // keep everything
  // rounding margin of the per-pixel evaluation (may_touch): relative to the largest term over the rect + absolute
  const float mx = fmaxf(fabsf(px - (float)(x0 * TILE_X)), fabsf((float)(x1 * TILE_X) - px));
  const float my = fmaxf(fabsf(py - (float)(y0 * TILE_Y)), fabsf((float)(y1 * TILE_Y) - py));
  const float taum = tau + 1e-5f * (A * mx * mx + C * my * my + 2.f * fabsf(B) * mx * my) + 1e-3f;
  const float idet = 1.0f / det, iA = 1.0f / A;
  const float hx = sqrtf(taum * C * idet), hy = sqrtf(taum * A * idet);
  if (!(hx < 1e6f && hy < 1e6f)) return all;
  const float dyx = -B * hx / C;  // dy of the ellipse's right-most point (the left-most one is at -dyx)
  const float D = det * iA, BA = B * iA;
  uint32_t mask = 0;
  for (int ty = y0; ty < y1; ty++) {
    const float lo = fmaxf((float)(ty * TILE_Y) - py, -hy), hi = fminf((float)min(ty * TILE_Y + TILE_Y - 1, H - 1) - py, hy);
    if (lo > hi) continue;  // the row's band misses the ellipse
    const float da = fminf(fmaxf(dyx, lo), hi), db = fminf(fmaxf(-dyx, lo), hi);
    const float xmax = -BA * da + sqrtf(fmaxf(0.f, (taum - D * da * da) * iA)) * 1.0001f + 0.01f;
    const float xmin = -BA * db - sqrtf(fmaxf(0.f, (taum - D * db * db) * iA)) * 1.0001f - 0.01f;
    // tiles whose pixel columns [16 tx, 16 tx + 15] meet [px + xmin, px + xmax]
    const int ta = max(x0, (int)ceilf((px + xmin - (float)(TILE_X - 1)) * (1.0f / TILE_X)));
    const int tb = min(x1 - 1, (int)floorf((px + xmax) * (1.0f / TILE_X)));
    if (ta > tb) continue;
    const int first = (ty - y0) * rw + (ta - x0), len = tb - ta + 1;
    mask |= (len >= 32 ? 0xffffffffu : ((1u << len) - 1u)) << first;
  }
  return mask & all;
}

// ---------------------------------------------------------------------------------------------
// K1: forward.cu:155-256
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(PRE_THREADS, 1024 / PRE_THREADS) k_preprocess_fwd(FwdArgs a, GeomView g, ImageView im) {
  extern __shared__ __align__(128) float sh_stage[];  // [256][3] f_dc rows, then [256][(M-1)*3] f_rest rows
  __shared__ __align__(8) unsigned long long sh_bar;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  int x0 = 0, y0 = 0, x1 = 0, y1 = 0;
  uint32_t tiles = 0, tmask = 0xffffffffu;  // rect area (the reference's tiles_touched) and which of those tiles are binned
  // whole CTA inside the array, coefficients beyond DC needed -> TMA staging
  const bool bulk = a.sh_bulk && a.D > 0 && (blockIdx.x + 1) * PRE_THREADS <= a.P;
  const int rest_row = (a.M - 1) * 3;
  if (bulk && threadIdx.x == 0) {
    const unsigned b_dc = PRE_THREADS * 3 * 4, b_rest = PRE_THREADS * rest_row * 4;
    bar_init_expect(&sh_bar, b_dc + b_rest);
    bulk_load(sh_stage, a.f_dc + (size_t)blockIdx.x * PRE_THREADS * 3, b_dc, &sh_bar);
    bulk_load(sh_stage + PRE_THREADS * 3, a.f_rest + (size_t)blockIdx.x * PRE_THREADS * rest_row, b_rest, &sh_bar);
  }
  if (bulk) __syncthreads();  // barrier initialised before anyone polls it
  const bool rows = a.sh_rows && a.D > 0 && (blockIdx.x + 1) * PRE_THREADS <= a.P;
  if (rows) {
    if (threadIdx.x == 0) {
      asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(&sh_bar)), "r"(PRE_THREADS) : "memory");
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    row_load(sh_stage + threadIdx.x * SH_ROW, a.shs + (size_t)idx * 48, 192, &sh_bar);
  }
  if (idx < a.P) {
    int radius_i = 0;
    const V3 p = {a.means3D[3 * idx], a.means3D[3 * idx + 1], a.means3D[3 * idx + 2]};
    // in_frustum (auxiliary.h:139-164): only the near plane is tested
    const V3 p_view = xf4x3(p, a.view);
    if (p_view.z <= 0.2f) {
      if (a.prefiltered) {
        printf("Point is filtered although prefiltered is set. This shouldn't happen!");
        __trap();
      }
    } else {
      const float4 p_hom = xf4x4(p, a.proj);
      const float p_w = 1.0f / (p_hom.w + 0.0000001f);
      const float ppx = p_hom.x * p_w, ppy = p_hom.y * p_w;
      float c3[6];
      if (a.cov3D_precomp != nullptr) {
#pragma unroll
        for (int k = 0; k < 6; k++) c3[k] = a.cov3D_precomp[6 * idx + k];
      } else {
        // computeCov3D, forward.cu:118-152
        const float mod = a.scale_modifier;
        float s0 = a.scales[3 * idx], s1 = a.scales[3 * idx + 1], s2 = a.scales[3 * idx + 2];
        float4 q = reinterpret_cast<const float4*>(a.rotations)[idx];
        if (a.fused) { s0 = expf(s0); s1 = expf(s1); s2 = expf(s2); q = act_normalize(q); }
        const Mat3 S = scale_mat(mod * s0, mod * s1, mod * s2);
        const Mat3 R = quat_mat(q.x, q.y, q.z, q.w);
        const Mat3 Mm = mmul(S, R);
        const Mat3 Sg = mmul(mtr(Mm), Mm);
        c3[0] = Sg.m[0][0]; c3[1] = Sg.m[0][1]; c3[2] = Sg.m[0][2];
        c3[3] = Sg.m[1][1]; c3[4] = Sg.m[1][2]; c3[5] = Sg.m[2][2];
#pragma unroll
        for (int k = 0; k < 6; k++) g.cov3D[6 * idx + k] = c3[k];
      }
      Cov2D cc;
      cov2d(p, a.focal_x, a.focal_y, a.tan_fovx, a.tan_fovy, c3, a.view, cc);
      const float cx = cc.cov.m[0][0], cy = cc.cov.m[0][1], cz = cc.cov.m[1][1];
      const float det = (cx * cz - cy * cy);
      if (det != 0.0f) {
        const float det_inv = 1.f / det;
        const float conA = cz * det_inv, conB = -cy * det_inv, conC = cx * det_inv;
        const float mid = 0.5f * (cx + cz);
        const float lambda1 = mid + sqrt(max(0.1f, mid * mid - det));
        const float lambda2 = mid - sqrt(max(0.1f, mid * mid - det));
        const float my_radius = ceil(3.f * sqrt(max(lambda1, lambda2)));
        const float px = ndc2pix(ppx, a.W), py = ndc2pix(ppy, a.H);
        tile_rect(px, py, (int)my_radius, a.gx, a.gy, x0, y0, x1, y1);
        if ((x1 - x0) * (y1 - y0) != 0) {
          float rgb[3];
          unsigned char cl = 0;
          if (a.colors_precomp == nullptr) {
            // computeColorFromSH, forward.cu:20-71 (coefficient stride M, degree D: quirk 13).  Written with
            // explicit mul / fma intrinsics in the contraction the reference's sm_90a SASS ends up with (ptxas
            // fuses its mul+add/sub pairs): weight_k rounded on its own, then res = fma(weight_k, sh_k, res).
            // coefficient 0 and coefficients >= 1 may live in two tensors (fused path: f_dc / f_rest)
            const float* sh0 = a.fused ? a.f_dc + (size_t)idx * 3 : a.shs + (size_t)idx * a.M * 3;
            const float* shr = a.fused ? a.f_rest + (size_t)idx * (a.M - 1) * 3 : sh0 + 3;
            if (bulk) {
              bar_wait0(&sh_bar);
              sh0 = sh_stage + threadIdx.x * 3;
              shr = sh_stage + PRE_THREADS * 3 + threadIdx.x * rest_row;
            } else if (rows) {
              bar_wait0(&sh_bar);
              sh0 = sh_stage + threadIdx.x * SH_ROW;
              shr = sh0 + 3;
            }
            const float ox = p.x - a.campos[0], oy = p.y - a.campos[1], oz = p.z - a.campos[2];
            const float len = sqrtf(__fmaf_rn(oz, oz, __fmaf_rn(ox, ox, __fmul_rn(oy, oy))));  // glm::length
            const float x = __fdiv_rn(ox, len), y = __fdiv_rn(oy, len), z = __fdiv_rn(oz, len);
            float w[16];
            int nco = 1;
            if (a.D > 0) {
              w[1] = -__fmul_rn(y, kC1); w[2] = __fmul_rn(z, kC1); w[3] = -__fmul_rn(x, kC1);
              nco = 4;
              if (a.D > 1) {
                const float xx = __fmul_rn(x, x), yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
                const float xy = __fmul_rn(x, y), yz = __fmul_rn(y, z), xz = __fmul_rn(x, z);
                const float zz2 = __fadd_rn(zz, zz), d = __fsub_rn(xx, yy);
                w[4] = __fmul_rn(xy, kC2[0]);
                w[5] = __fmul_rn(yz, kC2[1]);
                w[6] = __fmul_rn(__fsub_rn(__fsub_rn(zz2, xx), yy), kC2[2]);
                w[7] = __fmul_rn(xz, kC2[3]);
                w[8] = __fmul_rn(d, kC2[4]);
                nco = 9;
                if (a.D > 2) {
                  const float v = __fsub_rn(__fmaf_rn(zz, 4.0f, -xx), yy);  // 4zz - xx - yy
                  w[9] = __fmul_rn(__fmul_rn(y, kC3[0]), __fmaf_rn(xx, 3.0f, -yy));
                  w[10] = __fmul_rn(__fmul_rn(xy, kC3[1]), z);
                  w[11] = __fmul_rn(__fmul_rn(y, kC3[2]), v);
                  w[12] = __fmul_rn(__fmul_rn(z, kC3[3]), __fmaf_rn(yy, -3.0f, __fmaf_rn(xx, -3.0f, zz2)));
                  w[13] = __fmul_rn(__fmul_rn(x, kC3[4]), v);
                  w[14] = __fmul_rn(__fmul_rn(z, kC3[5]), d);
                  w[15] = __fmul_rn(__fmul_rn(x, kC3[6]), __fmaf_rn(yy, -3.0f, xx));
                  nco = 16;
                }
              }
            }
#pragma unroll
            for (int c = 0; c < 3; c++) {
              float res = __fmul_rn(sh0[c], kC0);
#pragma unroll
              for (int k = 1; k < 16; k++)
                if (k < nco) res = __fmaf_rn(w[k], shr[3 * (k - 1) + c], res);
              res = __fadd_rn(res, 0.5f);
              if (res < 0) cl |= (1u << c);
              rgb[c] = fmaxf(res, 0.0f);
            }
          } else {
            rgb[0] = a.colors_precomp[3 * idx]; rgb[1] = a.colors_precomp[3 * idx + 1]; rgb[2] = a.colors_precomp[3 * idx + 2];
          }
          radius_i = (int)my_radius;
          tiles = (uint32_t)((y1 - y0) * (x1 - x0));
          g.clamped[idx] = cl;
          float4* s = g.splat + (size_t)idx * SPLAT_F4;
          const float opac = a.fused ? act_sigmoid(a.opacities[idx]) : a.opacities[idx];
          // tau = 2 ln(255 o): alpha >= 1/255 needs the conic form <= tau (rectangle test of gsr_internal.cuh)
          const float4 r0 = make_float4(px, py, conA, conB), r1 = make_float4(conC, opac, p_view.z, rgb[0]);
          const float tau = 2.f * logf(255.f * opac);
          s[0] = r0;
          s[1] = r1;
          s[2] = make_float4(rgb[1], rgb[2], __int_as_float(idx), tau);
          // Exact tile culling: a (Gaussian, tile) pair of the reference's rect is binned only if the Gaussian can
          // reach alpha >= 1/255 on some pixel of that tile.  For every other pair the reference `continue`s on all
          // 256 pixels (forward.cu:353-355), so dropping it changes no output -- only the internal lists get shorter.
          if (tiles <= (uint32_t)kBigRect) tmask = tile_mask_of(px, py, conA, conB, conC, opac, tau, x0, y0, x1, y1, a.W, a.H);
        }
      }
    }
    if (tiles == 0) { x0 = y0 = x1 = y1 = 0; }
    g.radii[idx] = radius_i;
    if (a.radii_out) a.radii_out[idx] = radius_i;
    g.tiles_touched[idx] = tiles;
    g.tile_mask[idx] = tmask;
    g.rect[idx] = pack_rect(x0, y0, x1, y1);
  }
  // the reference's num_rendered (sum of the rect areas, rasterizer_impl.cu:280-284): one atomic per warp
  {
    const unsigned wsum = __reduce_add_sync(0xffffffffu, tiles);
    if ((threadIdx.x & 31) == 0 && wsum) atomicAdd(&im.hdr->num_rect, (unsigned long long)wsum);
  }
  // per-tile instance histogram (level 1 of the two-level binning; replaces InclusiveSum +
  // duplicateWithKeys offsets, rasterizer_impl.cu:280-300)
  const int T = a.gx * a.gy, warp_base = idx - (int)(threadIdx.x & 31);
  for_each_tile(x0, y0, x1, y1, tmask, a.gx, [&](int tile, unsigned src) {
    atomicAdd(&im.tile_count[subbin_of(warp_base + (int)src) * T + tile], 1u);
  });
  if ((bulk || rows) && threadIdx.x == 0) bar_wait0(&sh_bar);  // the copies must have landed before the CTA retires
}

// ---------------------------------------------------------------------------------------------
// K6 + K7 fused: backward.cu:144-274 then 346-412 (K6 assigns dL_dmean, K7 accumulates: quirk 7)
// ---------------------------------------------------------------------------------------------
// 36 warps per SM (<= 56 registers): as many CTAs as the 24.6-KB SH staging block of degree 3 lets an SM hold
__global__ void __launch_bounds__(PRE_THREADS, 1152 / PRE_THREADS) k_preprocess_bwd(BwdArgs a, GeomView g) {
  extern __shared__ __align__(128) float sh_stage[];  // SH rows in, SH gradient rows out (in place)
  __shared__ __align__(8) unsigned long long sh_bar;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int M = a.M;
  const bool bulk = a.sh_bulk && (blockIdx.x + 1) * PRE_THREADS <= a.P;
  const bool rows = a.sh_rows && (blockIdx.x + 1) * PRE_THREADS <= a.P;
  const int rest_row = (M - 1) * 3;
  if (rows && threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(&sh_bar)), "r"(PRE_THREADS) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (!bulk && !rows && idx >= a.P) return;
  const float4* ga = reinterpret_cast<const float4*>(g.grad + (size_t)idx * GRAD_F);
  float4 g0 = make_float4(0, 0, 0, 0), g1 = g0, g2 = g0;
  if (a.radii[idx] > 0) { g0 = ga[0]; g1 = ga[1]; g2 = ga[2]; }  // quirk 8
  // accumulator layout (written by the render backward): g0 = {dcol.r, dcol.g, dcol.b, ddepth},
  // g1 = {dopacity, sum u dx, sum u dy, sum u dx^2}, g2 = {sum u dx dy, sum u dy^2, -, -} with u = dL/dG * G per
  // (pixel, Gaussian) pair and d = mean2D - pixel.  G = exp(-(A dx^2 + C dy^2)/2 - B dx dy) gives
  //   dL/dmean2D = -(A Sx + B Sy, C Sy + B Sx) * (W/2, H/2)      (backward.cu:493-494, 598-599; quirk 6)
  //   dL/dconic  = -1/2 (Sxx, Sxy, Syy)                           (backward.cu:602-604)
  // Every output is linear in these ten sums.  A Gaussian the compositing never reached (no pair contributed, so no
  // sum moved off the memset's 0) gets all-zero gradients and reads nothing but its radius and accumulator: in a
  // dense scene most of them, because the pixels saturate before the rays are through it.
  const bool live = g0.x != 0.f || g0.y != 0.f || g0.z != 0.f || g0.w != 0.f || g1.x != 0.f || g1.y != 0.f ||
                    g1.z != 0.f || g1.w != 0.f || g2.x != 0.f || g2.y != 0.f;
  if (bulk) {  // SH of the warp's live rows only; the other rows are zeroed in place below
    const unsigned lm = __ballot_sync(0xffffffffu, live);
    const int w = threadIdx.x & ~31, w0 = blockIdx.x * PRE_THREADS + w;
    gather_live_rows(sh_stage + w * 3, a.f_dc + (size_t)w0 * 3, 12, lm);
    gather_live_rows(sh_stage + PRE_THREADS * 3 + w * rest_row, a.f_rest + (size_t)w0 * rest_row, rest_row * 4, lm);
  } else if (rows) {
    __syncthreads();  // barrier initialised
    if (live) row_load(sh_stage + threadIdx.x * SH_ROW, a.shs + (size_t)idx * 48, 192, &sh_bar);
    else bar_arrive(&sh_bar);
  }
  const float dL_dcolor[3] = {g0.x, g0.y, g0.z};
  const float dL_ddepth = g0.w, dL_dopac = g1.x;
  const float dcon_x = -0.5f * g1.w, dcon_y = -0.5f * g2.x, dcon_w = -0.5f * g2.y;

  float dm2x = 0.f, dm2y = 0.f, dop = 0.f;
  float dmean[3] = {0.f, 0.f, 0.f};
  float dcv[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  float dsc[3] = {0.f, 0.f, 0.f};
  float4 dq = make_float4(0.f, 0.f, 0.f, 0.f);
  V3 mean = {0.f, 0.f, 0.f};
  if (live) {
    mean = {a.means3D[3 * idx], a.means3D[3 * idx + 1], a.means3D[3 * idx + 2]};
    float c3[6];
    if (a.cov3D_precomp) {
#pragma unroll
      for (int k = 0; k < 6; k++) c3[k] = a.cov3D_precomp[6 * idx + k];
    } else {
      // recomputed with the forward's expressions (cheaper than reading back what it stored; backward_impl requires
      // scales and rotations here).  Written out rather than shared: moving the forward's copy into a helper keeps its
      // floating-point sequence but changes its register allocation.
      const float mod = a.scale_modifier;
      float s0 = a.scales[3 * idx], s1 = a.scales[3 * idx + 1], s2 = a.scales[3 * idx + 2];
      float4 q = reinterpret_cast<const float4*>(a.rotations)[idx];
      if (a.fused) { s0 = expf(s0); s1 = expf(s1); s2 = expf(s2); q = act_normalize(q); }
      const Mat3 S = scale_mat(mod * s0, mod * s1, mod * s2);
      const Mat3 R = quat_mat(q.x, q.y, q.z, q.w);
      const Mat3 Mm = mmul(S, R);
      const Mat3 Sg = mmul(mtr(Mm), Mm);
      c3[0] = Sg.m[0][0]; c3[1] = Sg.m[0][1]; c3[2] = Sg.m[0][2];
      c3[3] = Sg.m[1][1]; c3[4] = Sg.m[1][2]; c3[5] = Sg.m[2][2];
    }
    Cov2D cc;
    cov2d(mean, a.focal_x, a.focal_y, a.tan_fovx, a.tan_fovy, c3, a.view, cc);
    const float ca = cc.cov.m[0][0], cb = cc.cov.m[0][1], cd = cc.cov.m[1][1];
    const float det = ca * cd - cb * cb;  // != 0: the forward gave the Gaussian a radius
    {
      const float det_inv = 1.f / det;  // the forward's conic
      const float cA = cd * det_inv, cB = -cb * det_inv, cC = ca * det_inv;
      dm2x = -(cA * g1.y + cB * g1.z) * (float)(0.5 * a.W);
      dm2y = -(cC * g1.z + cB * g1.y) * (float)(0.5 * a.H);
    }
    // ---- K6 (backward.cu:144-274), derived in matrix form.  Notation (ordinary row/column math):
    //   cov2D = [[ca, cb], [cb, cd]] = A V A^T + 0.3 I,   A = J Wr (2x3),   conic = cov2D^-1,
    //   Gc = [[dcon_x, dcon_y], [dcon_y, dcon_w]]  (the compositing backward accumulates HALF of d/dB in dcon_y,
    //   so Gc is the symmetric gradient matrix as it stands).
    // d(conic) = -conic d(cov) conic  =>  dL/dcov2D = -conic Gc conic = -(adj Gc adj) / det^2, with the reference's
    // regularised 1 / (det^2 + 1e-7).
    const float kreg = 1.0f / ((det * det) + 0.0000001f);
    float S00 = 0.f, S01 = 0.f, S11 = 0.f;  // dL/dcov2D (symmetric; S01 is one off-diagonal entry)
    if (kreg != 0) {
      const float h0 = cd * dcon_x - cb * dcon_y, h1 = cd * dcon_y - cb * dcon_w;   // row 0 of adj * Gc
      const float h2 = ca * dcon_y - cb * dcon_x, h3 = ca * dcon_w - cb * dcon_y;   // row 1 of adj * Gc (times -1 col order)
      S00 = -kreg * (h0 * cd - h1 * cb);
      S01 = -kreg * (h1 * ca - h0 * cb);
      S11 = -kreg * (h3 * ca - h2 * cb);
    }
    float A2[2][3], Vs[3][3], Wr[3][3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
      A2[0][k] = cc.T.m[0][k]; A2[1][k] = cc.T.m[1][k];
#pragma unroll
      for (int j = 0; j < 3; j++) { Vs[k][j] = cc.Vrk.m[k][j]; Wr[k][j] = a.view[4 * j + k]; }
    }
    // dL/dV = A^T S A; the packed covariance stores every off-diagonal once, so those gradients count twice
    float SA[2][3];
#pragma unroll
    for (int k = 0; k < 3; k++) { SA[0][k] = S00 * A2[0][k] + S01 * A2[1][k]; SA[1][k] = S01 * A2[0][k] + S11 * A2[1][k]; }
    if (kreg != 0) {
      auto dV = [&](int k, int l) { return A2[0][k] * SA[0][l] + A2[1][k] * SA[1][l]; };
      dcv[0] = dV(0, 0); dcv[3] = dV(1, 1); dcv[5] = dV(2, 2);
      dcv[1] = 2.f * dV(0, 1); dcv[2] = 2.f * dV(0, 2); dcv[4] = 2.f * dV(1, 2);
    }
    // dL/dA = 2 S A V (V symmetric), dL/dJ = dL/dA Wr^T; J = [[fx/tz, 0, -fx tx/tz^2], [0, fy/tz, -fy ty/tz^2]]
    float dJ[2][3];
#pragma unroll
    for (int i = 0; i < 2; i++) {
      float dA[3];
#pragma unroll
      for (int j = 0; j < 3; j++) dA[j] = 2.f * (SA[i][0] * Vs[0][j] + SA[i][1] * Vs[1][j] + SA[i][2] * Vs[2][j]);
#pragma unroll
      for (int k = 0; k < 3; k++) dJ[i][k] = dA[0] * Wr[k][0] + dA[1] * Wr[k][1] + dA[2] * Wr[k][2];
    }
    const float itz = 1.f / cc.t.z, itz2 = itz * itz, itz3 = itz2 * itz;
    const float fx = a.focal_x, fy = a.focal_y;
    // the clamp of t.x / t.z, t.y / t.z to 1.3 tan(fov) gates the lateral gradients (backward.cu:188-191, 250-252)
    const bool clamp_x = cc.txtz < -cc.limx || cc.txtz > cc.limx, clamp_y = cc.tytz < -cc.limy || cc.tytz > cc.limy;
    const float dtx = clamp_x ? 0.f : -fx * itz2 * dJ[0][2];
    const float dty = clamp_y ? 0.f : -fy * itz2 * dJ[1][2];
    const float dtz = -fx * itz2 * dJ[0][0] - fy * itz2 * dJ[1][1] + (2.f * fx * cc.t.x) * itz3 * dJ[0][2] +
                      (2.f * fy * cc.t.y) * itz3 * dJ[1][2];
    const float* vm = a.view;
    // t = Wr p + translation  =>  dL/dp = Wr^T dL/dt   (K6 ASSIGNS the mean gradient, K7 accumulates: quirk 7)
#pragma unroll
    for (int j = 0; j < 3; j++) dmean[j] = Wr[0][j] * dtx + Wr[1][j] * dty + Wr[2][j] * dtz;

    // ---- K7 (backward.cu:346-412)
    const float* proj = a.proj;
    const float4 m_hom = xf4x4(mean, proj);
    const float m_w = 1.0f / (m_hom.w + 0.0000001f);
    const float mul1 = (proj[0] * mean.x + proj[4] * mean.y + proj[8] * mean.z + proj[12]) * m_w * m_w;
    const float mul2 = (proj[1] * mean.x + proj[5] * mean.y + proj[9] * mean.z + proj[13]) * m_w * m_w;
    dmean[0] += (proj[0] * m_w - proj[3] * mul1) * dm2x + (proj[1] * m_w - proj[3] * mul2) * dm2y;
    dmean[1] += (proj[4] * m_w - proj[7] * mul1) * dm2x + (proj[5] * m_w - proj[7] * mul2) * dm2y;
    dmean[2] += (proj[8] * m_w - proj[11] * mul1) * dm2x + (proj[9] * m_w - proj[11] * mul2) * dm2y;
    const float mul3 = vm[2] * mean.x + vm[6] * mean.y + vm[10] * mean.z + vm[14];
    dmean[0] += (vm[2] - vm[3] * mul3) * dL_ddepth;
    dmean[1] += (vm[6] - vm[7] * mul3) * dL_ddepth;
    dmean[2] += (vm[10] - vm[11] * mul3) * dL_ddepth;

    if (a.scales) {
      // cov3D backward (backward.cu:278-341), derived in matrix form: Sigma = N N^T with N = R diag(s), R the standard
      // rotation matrix of the quaternion AS GIVEN (no normalisation Jacobian: quirk 2), s = scale_modifier * scale.
      //   dL/dN = 2 dSigma N  (dSigma symmetric: the packed off-diagonal gradients are split in two halves)
      //   dL/ds_i = sum_r dN[r][i] R[r][i]   (taken w.r.t. the modified scale, like the reference)
      //   dL/dR[r][i] = dN[r][i] s_i, then through the nine entries of R(q).
      // (read again rather than kept in registers through K6 / K7: the second read hits L1)
      float4 q = reinterpret_cast<const float4*>(a.rotations)[idx];
      float as0 = a.scales[3 * idx], as1 = a.scales[3 * idx + 1], as2 = a.scales[3 * idx + 2];
      float inv_n = 0.f;
      if (a.fused) { q = act_normalize(q, &inv_n); as0 = expf(as0); as1 = expf(as1); as2 = expf(as2); }
      const float r = q.x, x = q.y, y = q.z, z = q.w;
      const float Rq[3][3] = {{1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (x * z + r * y)},
                              {2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - r * x)},
                              {2.f * (x * z - r * y), 2.f * (y * z + r * x), 1.f - 2.f * (x * x + y * y)}};
      const float sv[3] = {a.scale_modifier * as0, a.scale_modifier * as1, a.scale_modifier * as2};
      const float dSg[3][3] = {{dcv[0], 0.5f * dcv[1], 0.5f * dcv[2]},
                               {0.5f * dcv[1], dcv[3], 0.5f * dcv[4]},
                               {0.5f * dcv[2], 0.5f * dcv[4], dcv[5]}};
      float dR[3][3];
#pragma unroll
      for (int i = 0; i < 3; i++) {
        float acc = 0.f;
#pragma unroll
        for (int rr = 0; rr < 3; rr++) {
          // dN[rr][i] = 2 sum_m dSigma[rr][m] N[m][i],  N[m][i] = R[m][i] s_i
          const float dN = 2.f * sv[i] * (dSg[rr][0] * Rq[0][i] + dSg[rr][1] * Rq[1][i] + dSg[rr][2] * Rq[2][i]);
          acc += dN * Rq[rr][i];
          dR[rr][i] = dN * sv[i];
        }
        dsc[i] = acc;
      }
      dq.x = 2.f * (z * (dR[1][0] - dR[0][1]) + y * (dR[0][2] - dR[2][0]) + x * (dR[2][1] - dR[1][2]));
      dq.y = 2.f * (y * (dR[0][1] + dR[1][0]) + z * (dR[0][2] + dR[2][0]) + r * (dR[2][1] - dR[1][2])) - 4.f * x * (dR[1][1] + dR[2][2]);
      dq.z = 2.f * (x * (dR[0][1] + dR[1][0]) + r * (dR[0][2] - dR[2][0]) + z * (dR[1][2] + dR[2][1])) - 4.f * y * (dR[0][0] + dR[2][2]);
      dq.w = 2.f * (r * (dR[1][0] - dR[0][1]) + x * (dR[0][2] + dR[2][0]) + y * (dR[1][2] + dR[2][1])) - 4.f * z * (dR[0][0] + dR[1][1]);
      if (a.fused) {
        // chain through exp (scale) and F.normalize (rotation): d/dq_raw = (g - qhat (qhat . g)) / |q_raw|
        dsc[0] *= as0; dsc[1] *= as1; dsc[2] *= as2;
        const float dot = q.x * dq.x + q.y * dq.y + q.z * dq.z + q.w * dq.w;
        dq = make_float4((dq.x - q.x * dot) * inv_n, (dq.y - q.y * dot) * inv_n, (dq.z - q.z * dot) * inv_n,
                         (dq.w - q.w * dot) * inv_n);
      }
    }
    if (a.fused) {
      const float so = act_sigmoid(a.opacities_raw[idx]);
      dop = dL_dopac * so * (1.0f - so);  // through sigmoid
    } else {
      dop = dL_dopac;
    }
  }
  // everything but the mean gradient is final: stored before the SH part, which only adds to dmean
  a.dL_dmean2D[3 * idx] = dm2x; a.dL_dmean2D[3 * idx + 1] = dm2y; a.dL_dmean2D[3 * idx + 2] = 0.f;
  a.dL_dopacity[idx] = dop;
  if (a.dL_dcolor) {
    a.dL_dcolor[3 * idx] = dL_dcolor[0]; a.dL_dcolor[3 * idx + 1] = dL_dcolor[1]; a.dL_dcolor[3 * idx + 2] = dL_dcolor[2];
  }
  if (a.dL_dconic) reinterpret_cast<float4*>(a.dL_dconic)[idx] = make_float4(dcon_x, dcon_y, 0.f, dcon_w);
  if (a.dL_ddepth) a.dL_ddepth[idx] = dL_ddepth;
  if (a.dL_dcov3D) {
#pragma unroll
    for (int k = 0; k < 6; k++) a.dL_dcov3D[6 * idx + k] = dcv[k];
  }
  a.dL_dscale[3 * idx] = dsc[0]; a.dL_dscale[3 * idx + 1] = dsc[1]; a.dL_dscale[3 * idx + 2] = dsc[2];
  reinterpret_cast<float4*>(a.dL_drot)[idx] = dq;

  // SH gradient destinations: one [P,M,3] tensor, or the f_dc / f_rest pair of the fused variant
  float* dsh0 = a.fused ? a.dL_df_dc + (size_t)idx * 3 : (a.dL_dsh ? a.dL_dsh + (size_t)idx * M * 3 : nullptr);
  float* dshr = a.fused ? a.dL_df_rest + (size_t)idx * (M - 1) * 3 : (dsh0 ? dsh0 + 3 : nullptr);
  if (bulk) {  // gradients are written over the staged coefficients and leave with a bulk store
    asm volatile("cp.async.wait_all;" ::: "memory");
    __syncwarp();  // the warp's chunks have landed (a chunk may straddle two lanes' rows)
    dsh0 = sh_stage + threadIdx.x * 3;
    dshr = sh_stage + PRE_THREADS * 3 + threadIdx.x * rest_row;
  } else if (rows) {
    bar_wait0(&sh_bar);
    dsh0 = sh_stage + threadIdx.x * SH_ROW;
    dshr = dsh0 + 3;
  }
  auto dsh_zero = [&](int from) {
    if (!dsh0) return;
    if (from == 0) { dsh0[0] = 0.f; dsh0[1] = 0.f; dsh0[2] = 0.f; from = 1; }
    for (int k = from; k < M; k++) { dshr[3 * (k - 1)] = 0.f; dshr[3 * (k - 1) + 1] = 0.f; dshr[3 * (k - 1) + 2] = 0.f; }
  };
  if (live && (a.fused || a.shs != nullptr)) {
    // SH backward, backward.cu:20-139
    const float* sh0 = (bulk || rows) ? dsh0 : (a.fused ? a.f_dc + (size_t)idx * 3 : a.shs + (size_t)idx * M * 3);
    const float* shr = (bulk || rows) ? dshr : (a.fused ? a.f_rest + (size_t)idx * (M - 1) * 3 : sh0 + 3);
    const float ox = mean.x - a.campos[0], oy = mean.y - a.campos[1], oz = mean.z - a.campos[2];
    const float len = sqrt(ox * ox + oy * oy + oz * oz);
    const float x = ox / len, y = oy / len, z = oz / len;
    const unsigned char cl = g.clamped[idx];
    float dRGB[3];
#pragma unroll
    for (int c = 0; c < 3; c++) dRGB[c] = dL_dcolor[c] * ((cl >> c) & 1 ? 0.f : 1.f);
    float ddx = 0.f, ddy = 0.f, ddz = 0.f;
    auto emit = [&](int k, float w, float bx, float by, float bz) {
      // dL_dsh[k] = w * dRGB ; d(dir) += d(basis_k)/d(dir) * dot(sh[k], dRGB)
      const float* shk = k == 0 ? sh0 : shr + 3 * (k - 1);
      float* dk = k == 0 ? dsh0 : dshr + 3 * (k - 1);
      const float s = shk[0] * dRGB[0] + shk[1] * dRGB[1] + shk[2] * dRGB[2];
      dk[0] = w * dRGB[0]; dk[1] = w * dRGB[1]; dk[2] = w * dRGB[2];
      ddx += bx * s; ddy += by * s; ddz += bz * s;
    };
    emit(0, kC0, 0.f, 0.f, 0.f);
    int used = 1;
    if (a.D > 0) {
      emit(1, -kC1 * y, 0.f, -kC1, 0.f);
      emit(2, kC1 * z, 0.f, 0.f, kC1);
      emit(3, -kC1 * x, -kC1, 0.f, 0.f);
      used = 4;
      if (a.D > 1) {
        const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
        emit(4, kC2[0] * xy, kC2[0] * y, kC2[0] * x, 0.f);
        emit(5, kC2[1] * yz, 0.f, kC2[1] * z, kC2[1] * y);
        emit(6, kC2[2] * (2.f * zz - xx - yy), kC2[2] * 2.f * -x, kC2[2] * 2.f * -y, kC2[2] * 2.f * 2.f * z);
        emit(7, kC2[3] * xz, kC2[3] * z, 0.f, kC2[3] * x);
        emit(8, kC2[4] * (xx - yy), kC2[4] * 2.f * x, kC2[4] * 2.f * -y, 0.f);
        used = 9;
        if (a.D > 2) {
          emit(9, kC3[0] * y * (3.f * xx - yy), kC3[0] * 3.f * 2.f * xy, kC3[0] * 3.f * (xx - yy), 0.f);
          emit(10, kC3[1] * xy * z, kC3[1] * yz, kC3[1] * xz, kC3[1] * xy);
          emit(11, kC3[2] * y * (4.f * zz - xx - yy), kC3[2] * -2.f * xy, kC3[2] * (-3.f * yy + 4.f * zz - xx), kC3[2] * 4.f * 2.f * yz);
          emit(12, kC3[3] * z * (2.f * zz - 3.f * xx - 3.f * yy), kC3[3] * -3.f * 2.f * xz, kC3[3] * -3.f * 2.f * yz, kC3[3] * 3.f * (2.f * zz - xx - yy));
          emit(13, kC3[4] * x * (4.f * zz - xx - yy), kC3[4] * (-3.f * xx + 4.f * zz - yy), kC3[4] * -2.f * xy, kC3[4] * 4.f * 2.f * xz);
          emit(14, kC3[5] * z * (xx - yy), kC3[5] * 2.f * xz, kC3[5] * -2.f * yz, kC3[5] * (xx - yy));
          emit(15, kC3[6] * x * (xx - 3.f * yy), kC3[6] * 3.f * (xx - yy), kC3[6] * -3.f * 2.f * xy, 0.f);
          used = 16;
        }
      }
    }
    dsh_zero(used);
    // dnormvdv (auxiliary.h:107-117)
    const float sum2 = ox * ox + oy * oy + oz * oz;
    const float invsum32 = 1.0f / sqrt(sum2 * sum2 * sum2);
    dmean[0] += ((+sum2 - ox * ox) * ddx - oy * ox * ddy - oz * ox * ddz) * invsum32;
    dmean[1] += (-ox * oy * ddx + (sum2 - oy * oy) * ddy - oz * oy * ddz) * invsum32;
    dmean[2] += (-ox * oz * ddx - oy * oz * ddy + (sum2 - oz * oz) * ddz) * invsum32;
  } else {
    dsh_zero(0);
  }
  a.dL_dmean3D[3 * idx] = dmean[0]; a.dL_dmean3D[3 * idx + 1] = dmean[1]; a.dL_dmean3D[3 * idx + 2] = dmean[2];
  if (bulk) {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> visible to the TMA engine
    __syncthreads();
    if (threadIdx.x == 0) {
      bulk_store(a.dL_df_dc + (size_t)blockIdx.x * PRE_THREADS * 3, sh_stage, PRE_THREADS * 3 * 4);
      bulk_store(a.dL_df_rest + (size_t)blockIdx.x * PRE_THREADS * rest_row, sh_stage + PRE_THREADS * 3,
                 PRE_THREADS * rest_row * 4);
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // shared memory may be released after this
    }
  } else if (rows) {
    // each thread ships the gradient row it wrote itself: its own generic-proxy writes -> async proxy
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    bulk_store(a.dL_dsh + (size_t)idx * 48, sh_stage + threadIdx.x * SH_ROW, 192);
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
  }
}

// checkFrustum, rasterizer_impl.cu:54-66
__global__ void k_mark_visible(int P, const float* __restrict__ means3D, const float* __restrict__ view,
                               unsigned char* __restrict__ present) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= P) return;
  const V3 p = {means3D[3 * idx], means3D[3 * idx + 1], means3D[3 * idx + 2]};
  present[idx] = xf4x3(p, view).z > 0.2f;
}

}  // namespace

void launch_preprocess_fwd(const FwdArgs& a, GeomView g, ImageView im, cudaStream_t st) {
  const size_t smem = a.sh_bulk ? (size_t)PRE_THREADS * a.M * 12 : (a.sh_rows ? (size_t)PRE_THREADS * SH_ROW * 4 : 0);
  const DeviceInfo& di = device_info();
  if (smem > di.pre_fwd_smem) {  // opt in once per device (again only if a larger staging block shows up)
    cudaFuncSetAttribute(k_preprocess_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    di.pre_fwd_smem = smem;
  }
  launch_high_priority(k_preprocess_fwd, dim3((a.P + PRE_THREADS - 1) / PRE_THREADS), dim3(PRE_THREADS), smem, st, a, g, im);
}
void launch_preprocess_bwd(const BwdArgs& a, GeomView g, cudaStream_t st) {
  const size_t smem = a.sh_bulk ? (size_t)PRE_THREADS * a.M * 12 : (a.sh_rows ? (size_t)PRE_THREADS * SH_ROW * 4 : 0);
  const DeviceInfo& di = device_info();
  if (smem > di.pre_bwd_smem) {
    cudaFuncSetAttribute(k_preprocess_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    di.pre_bwd_smem = smem;
  }
  launch_high_priority(k_preprocess_bwd, dim3((a.P + PRE_THREADS - 1) / PRE_THREADS), dim3(PRE_THREADS), smem, st, a, g);
}
void launch_mark_visible(int P, const float* means3D, const float* view, const float*, unsigned char* present,
                         cudaStream_t st) {
  k_mark_visible<<<(P + 255) / 256, 256, 0, st>>>(P, means3D, view, present);
}

}  // namespace gsr
