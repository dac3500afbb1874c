// Surfel (2D Gaussian) rasterizer: projection, compositing forward / backward, projection backward, and the C ABI entry
// points gsr_surfel_* of include/gsr.h.  The contract (ray-splat intersection through the per-splat T matrix, the
// screen-space low-pass filter, depth / normal / distortion / median maps) is written down in DESIGN.md §3, surfel rasterizer.
//
// The binning is the 3DGS path's, unchanged: the projection kernel writes the fields k_tile_scan, k_scatter and
// k_tile_sort read (packed tile rect, tile mask, depth key at float 6 of a 48-byte record, sub-binned tile histogram),
// so a GeomView whose `splat` is the first half of the surfel record drives them.  No exact tile culling: every tile of
// the rect is binned.
#include "../../include/gsr.h"
#include "gsr_internal.cuh"

namespace gsr {

namespace {

constexpr float kNear = 0.2f, kFar = 100.f;
constexpr int SURF_GRAD = 20;  // per-Gaussian accumulator: mean2D 2, Tu 3, Tv 3, Tw 3, n_view 3, opacity 1, rgb 3 (18 used)
constexpr int REC_A = 3, REC_B = 2;  // float4s per Gaussian in the two record arrays
constexpr int SURF_THREADS = 128;
constexpr int CB = 256;  // records staged per batch of the compositing kernels (one per thread of the 16x16 CTA)

// Surfel geometry buffer.  Record (80 B, two arrays so that the first one has the 48-byte stride the binning reads):
//   A[0] = { mean2D.x, mean2D.y, Tw.x, Tw.y }   A[1] = { Tw.z, opacity, view depth (sort key), bits(index) }
//   A[2] = { Tu.x, Tu.y, Tu.z, Tv.x }           B[0] = { Tv.y, Tv.z, n_view.x, n_view.y }   B[1] = { n_view.z, rgb }
struct SurfGeom {
  float4* recA;            // [P][3]
  float4* recB;            // [P][2]
  uint2* rect;             // [P] packed tile rect
  uint32_t* tile_mask;     // [P] every tile of a rect of <= 32 tiles
  int* radii;              // [P]
  unsigned char* clamped;  // [P] bit c: SH colour channel c was clamped at 0
  float* grad;             // [P][SURF_GRAD] compositing-backward accumulator
};
// Surfel image buffer: the 3DGS ImageView (header, final_T, n_contrib, tile histogram / ranges / cursors, ...) followed
// by what the distortion and median gradients need per pixel.
struct SurfImage {
  ImageView im;
  float *M1, *M2;   // [H*W] final sums of w*m and w*m^2 (distortion)
  uint32_t* med_c;  // [H*W] 1 + position in the tile list of the median splat; 0: none
};

SurfGeom carve_sgeom(char* base, int P) {
  SurfGeom g;
  char* p = base;
  take(p, g.recA, (size_t)P * REC_A);
  take(p, g.recB, (size_t)P * REC_B);
  take(p, g.rect, (size_t)P);
  take(p, g.tile_mask, (size_t)P);
  take(p, g.radii, (size_t)P);
  take(p, g.clamped, (size_t)P);
  take(p, g.grad, (size_t)P * SURF_GRAD);
  return g;
}
size_t sgeom_bytes(int P) {
  SurfGeom g = carve_sgeom(nullptr, P);
  return reinterpret_cast<size_t>(g.grad + (size_t)P * SURF_GRAD) + 512;
}
SurfImage carve_simage(char* base, int W, int H) {
  SurfImage s;
  s.im = carve_image(base, W, H);
  char* p = base + image_bytes(W, H);
  const size_t N = (size_t)W * H;
  take(p, s.M1, N);
  take(p, s.M2, N);
  take(p, s.med_c, N);
  return s;
}
size_t simage_bytes(int W, int H) {
  SurfImage s = carve_simage(nullptr, W, H);
  return reinterpret_cast<size_t>(s.med_c + (size_t)W * H) + 512;
}
// what the binning kernels read, pointed at the surfel buffer
GeomView binning_view(const SurfGeom& s) {
  GeomView g{};
  g.splat = s.recA;
  g.rect = s.rect;
  g.tile_mask = s.tile_mask;
  g.radii = s.radii;
  return g;
}

struct SurfArgs {
  int P, D, M, W, H, gx, gy;
  const float *means3D, *shs, *colors_precomp, *opacities, *scales, *rotations, *view, *proj, *campos;
  float mod;
  int* radii_out;
};

// ---- device helpers ------------------------------------------------------------------------------------------------
struct F3 { float x, y, z; };
__device__ __forceinline__ F3 cross3(F3 a, F3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
__device__ __forceinline__ float dot3(F3 a, F3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

// Rotation matrix of the quaternion (w, x, y, z), R[row][col]; the splat's tangent axes are columns 0 and 1, its normal
// column 2.
__device__ __forceinline__ void rotmat(float4 q, float R[3][3]) {
  const float w = q.x, x = q.y, y = q.z, z = q.w;
  R[0][0] = 1.f - 2.f * (y * y + z * z); R[0][1] = 2.f * (x * y - w * z);       R[0][2] = 2.f * (x * z + w * y);
  R[1][0] = 2.f * (x * y + w * z);       R[1][1] = 1.f - 2.f * (x * x + z * z); R[1][2] = 2.f * (y * z - w * x);
  R[2][0] = 2.f * (x * z - w * y);       R[2][1] = 2.f * (y * z + w * x);       R[2][2] = 1.f - 2.f * (x * x + y * y);
}

// Per-Gaussian geometry of the contract (DESIGN.md §3, surfel rasterizer): T matrix, camera-facing view normal, screen box.
struct SurfProj {
  F3 pv;              // view-space centre
  float R[3][3];
  float su, sv;       // scales * scale_modifier
  F3 Tu, Tv, Tw;
  F3 nv;              // view-space normal, facing the camera
  float sign;         // the flip applied to the rotated normal (held constant by the backward)
  float d, mx, my, radius;
};
__device__ __forceinline__ bool surfel_project(int idx, const float* __restrict__ means3D, const float* __restrict__ scales,
                                               const float* __restrict__ rotations, float mod,
                                               const float* __restrict__ view, const float* __restrict__ proj, int W,
                                               int H, SurfProj& s) {
  const float p[3] = {means3D[3 * idx], means3D[3 * idx + 1], means3D[3 * idx + 2]};
  s.pv = {view[0] * p[0] + view[4] * p[1] + view[8] * p[2] + view[12],
          view[1] * p[0] + view[5] * p[1] + view[9] * p[2] + view[13],
          view[2] * p[0] + view[6] * p[1] + view[10] * p[2] + view[14]};
  if (s.pv.z <= kNear) return false;
  rotmat(reinterpret_cast<const float4*>(rotations)[idx], s.R);
  s.su = scales[2 * idx] * mod;
  s.sv = scales[2 * idx + 1] * mod;
  // clip coordinates of the tangent axes (w = 0) and of the centre (w = 1): c = [X, 1] @ projmatrix
  float cu[4], cv[4], cp[4];
#pragma unroll
  for (int c = 0; c < 4; c++) {
    cu[c] = (s.R[0][0] * proj[c] + s.R[1][0] * proj[4 + c] + s.R[2][0] * proj[8 + c]) * s.su;
    cv[c] = (s.R[0][1] * proj[c] + s.R[1][1] * proj[4 + c] + s.R[2][1] * proj[8 + c]) * s.sv;
    cp[c] = p[0] * proj[c] + p[1] * proj[4 + c] + p[2] * proj[8 + c] + proj[12 + c];
  }
  // pixel-homogeneous rows (ndc2Pix): hx = W/2 c.x + (W-1)/2 c.w, hy = H/2 c.y + (H-1)/2 c.w, hw = c.w
  const float aW = 0.5f * W, bW = 0.5f * (W - 1), aH = 0.5f * H, bH = 0.5f * (H - 1);
  s.Tu = {aW * cu[0] + bW * cu[3], aW * cv[0] + bW * cv[3], aW * cp[0] + bW * cp[3]};
  s.Tv = {aH * cu[1] + bH * cu[3], aH * cv[1] + bH * cv[3], aH * cp[1] + bH * cp[3]};
  s.Tw = {cu[3], cv[3], cp[3]};
  const F3 nr = {view[0] * s.R[0][2] + view[4] * s.R[1][2] + view[8] * s.R[2][2],
                 view[1] * s.R[0][2] + view[5] * s.R[1][2] + view[9] * s.R[2][2],
                 view[2] * s.R[0][2] + view[6] * s.R[1][2] + view[10] * s.R[2][2]};
  const float facing = dot3(nr, s.pv);
  if (facing == 0.f) return false;
  s.sign = facing > 0.f ? -1.f : 1.f;
  s.nv = {s.sign * nr.x, s.sign * nr.y, s.sign * nr.z};
  // screen box, cutoff 3: Q = diag(9, 9, -1)
  s.d = 9.f * s.Tw.x * s.Tw.x + 9.f * s.Tw.y * s.Tw.y - s.Tw.z * s.Tw.z;
  if (s.d == 0.f) return false;
  s.mx = (9.f * s.Tu.x * s.Tw.x + 9.f * s.Tu.y * s.Tw.y - s.Tu.z * s.Tw.z) / s.d;
  s.my = (9.f * s.Tv.x * s.Tw.x + 9.f * s.Tv.y * s.Tw.y - s.Tv.z * s.Tw.z) / s.d;
  const float hx = sqrtf(fmaxf(1e-4f, s.mx * s.mx - (9.f * s.Tu.x * s.Tu.x + 9.f * s.Tu.y * s.Tu.y - s.Tu.z * s.Tu.z) / s.d));
  const float hy = sqrtf(fmaxf(1e-4f, s.my * s.my - (9.f * s.Tv.x * s.Tv.x + 9.f * s.Tv.y * s.Tv.y - s.Tv.z * s.Tv.z) / s.d));
  s.radius = ceilf(fmaxf(fmaxf(hx, hy), 3.f * 0.707106f));
  // a non-finite box (degenerate input) culls, as does one too large for the integer rect arithmetic
  return isfinite(s.mx) && isfinite(s.my) && s.radius < 1e7f;
}

// SH basis (the 3DGS path's constants and ordering)
__device__ __forceinline__ int sh_basis(int D, F3 d, float w[16], F3 gw[16]) {
  constexpr float C0 = 0.28209479177387814f, C1 = 0.4886025119029199f;
  constexpr float C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f, -1.0925484305920792f,
                           0.5462742152960396f};
  constexpr float C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f, 0.3731763325901154f,
                           -0.4570457994644658f, 1.445305721320277f, -0.5900435899266435f};
  const float x = d.x, y = d.y, z = d.z;
  w[0] = C0; gw[0] = {0.f, 0.f, 0.f};
  if (D < 1) return 1;
  w[1] = -C1 * y; gw[1] = {0.f, -C1, 0.f};
  w[2] = C1 * z;  gw[2] = {0.f, 0.f, C1};
  w[3] = -C1 * x; gw[3] = {-C1, 0.f, 0.f};
  if (D < 2) return 4;
  const float xx = x * x, yy = y * y, zz = z * z;
  w[4] = C2[0] * x * y;                 gw[4] = {C2[0] * y, C2[0] * x, 0.f};
  w[5] = C2[1] * y * z;                 gw[5] = {0.f, C2[1] * z, C2[1] * y};
  w[6] = C2[2] * (2.f * zz - xx - yy);  gw[6] = {-2.f * C2[2] * x, -2.f * C2[2] * y, 4.f * C2[2] * z};
  w[7] = C2[3] * x * z;                 gw[7] = {C2[3] * z, 0.f, C2[3] * x};
  w[8] = C2[4] * (xx - yy);             gw[8] = {2.f * C2[4] * x, -2.f * C2[4] * y, 0.f};
  if (D < 3) return 9;
  w[9] = C3[0] * y * (3.f * xx - yy);        gw[9] = {C3[0] * 6.f * x * y, C3[0] * (3.f * xx - 3.f * yy), 0.f};
  w[10] = C3[1] * x * y * z;                 gw[10] = {C3[1] * y * z, C3[1] * x * z, C3[1] * x * y};
  w[11] = C3[2] * y * (4.f * zz - xx - yy);  gw[11] = {-2.f * C3[2] * x * y, C3[2] * (4.f * zz - xx - 3.f * yy), 8.f * C3[2] * y * z};
  w[12] = C3[3] * z * (2.f * zz - 3.f * xx - 3.f * yy);
  gw[12] = {-6.f * C3[3] * x * z, -6.f * C3[3] * y * z, C3[3] * (6.f * zz - 3.f * xx - 3.f * yy)};
  w[13] = C3[4] * x * (4.f * zz - xx - yy);  gw[13] = {C3[4] * (4.f * zz - 3.f * xx - yy), -2.f * C3[4] * x * y, 8.f * C3[4] * x * z};
  w[14] = C3[5] * z * (xx - yy);             gw[14] = {2.f * C3[5] * x * z, -2.f * C3[5] * y * z, C3[5] * (xx - yy)};
  w[15] = C3[6] * x * (xx - 3.f * yy);       gw[15] = {C3[6] * (3.f * xx - 3.f * yy), -6.f * C3[6] * x * y, 0.f};
  return 16;
}
__device__ __forceinline__ F3 view_dir(int idx, const float* __restrict__ means3D, const float* __restrict__ campos, float& len) {
  const F3 o = {means3D[3 * idx] - campos[0], means3D[3 * idx + 1] - campos[1], means3D[3 * idx + 2] - campos[2]};
  len = sqrtf(dot3(o, o));
  return {o.x / len, o.y / len, o.z / len};
}

// One (pixel, splat) pair, shared by the two compositing kernels so that both take the same decisions: ray-splat
// intersection s (splat-plane coordinates of the pixel's ray), rho3 = |s|^2, the low-pass distance rho2, and the depth.
// False: the splat is skipped at this pixel (parallel ray or depth in front of the near plane).
struct Pair { F3 k, l, p; float sx, sy, rho3, rho2, z; };
__device__ __forceinline__ bool eval_pair(float fx, float fy, float mx, float my, F3 Tu, F3 Tv, F3 Tw, Pair& q) {
  q.k = {fx * Tw.x - Tu.x, fx * Tw.y - Tu.y, fx * Tw.z - Tu.z};
  q.l = {fy * Tw.x - Tv.x, fy * Tw.y - Tv.y, fy * Tw.z - Tv.z};
  q.p = cross3(q.k, q.l);
  if (q.p.z == 0.f) return false;
  q.sx = q.p.x / q.p.z;
  q.sy = q.p.y / q.p.z;
  q.rho3 = q.sx * q.sx + q.sy * q.sy;
  const float dx = mx - fx, dy = my - fy;
  q.rho2 = 2.f * (dx * dx + dy * dy);
  q.z = q.rho3 <= q.rho2 ? q.sx * Tw.x + q.sy * Tw.y + Tw.z : Tw.z;
  return !(q.z < kNear);
}
__device__ __forceinline__ float pair_gauss(const Pair& q) { return expf(-0.5f * fminf(q.rho3, q.rho2)); }
// distortion's normalised depth m(z) and dm/dz
__device__ __forceinline__ float dist_m(float z) { return kFar / (kFar - kNear) * (1.f - kNear / z); }
__device__ __forceinline__ float dist_dm(float z) { return kFar / (kFar - kNear) * kNear / (z * z); }

// ---- projection forward --------------------------------------------------------------------------------------------
// 10 CTAs per SM: keeps the kernel at 48 registers (the shared tile walk alone would let ptxas take 50, and 9 CTAs)
__global__ void __launch_bounds__(SURF_THREADS, 10) k_surfel_project(SurfArgs a, SurfGeom g, ImageView im) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  int x0 = 0, y0 = 0, x1 = 0, y1 = 0;
  uint32_t tiles = 0, tmask = 0;
  if (idx < a.P) {
    int radius_i = 0;
    SurfProj s;
    if (surfel_project(idx, a.means3D, a.scales, a.rotations, a.mod, a.view, a.proj, a.W, a.H, s)) {
      tile_rect(s.mx, s.my, (int)s.radius, a.gx, a.gy, x0, y0, x1, y1);
      if ((x1 - x0) * (y1 - y0) != 0) {
        float rgb[3];
        unsigned char cl = 0;
        if (a.colors_precomp == nullptr) {
          float len, w[16];
          F3 gw[16];
          const int nco = sh_basis(a.D, view_dir(idx, a.means3D, a.campos, len), w, gw);
          const float* sh = a.shs + (size_t)idx * a.M * 3;
#pragma unroll
          for (int c = 0; c < 3; c++) {
            float r = 0.f;
            for (int k = 0; k < nco; k++) r += w[k] * sh[3 * k + c];
            r += 0.5f;
            if (r < 0.f) cl |= (unsigned char)(1u << c);
            rgb[c] = fmaxf(r, 0.f);
          }
        } else {
          rgb[0] = a.colors_precomp[3 * idx]; rgb[1] = a.colors_precomp[3 * idx + 1]; rgb[2] = a.colors_precomp[3 * idx + 2];
        }
        g.clamped[idx] = cl;
        float4* A = g.recA + (size_t)idx * REC_A;
        float4* B = g.recB + (size_t)idx * REC_B;
        A[0] = make_float4(s.mx, s.my, s.Tw.x, s.Tw.y);
        A[1] = make_float4(s.Tw.z, a.opacities[idx], s.pv.z, __int_as_float(idx));
        A[2] = make_float4(s.Tu.x, s.Tu.y, s.Tu.z, s.Tv.x);
        B[0] = make_float4(s.Tv.y, s.Tv.z, s.nv.x, s.nv.y);
        B[1] = make_float4(s.nv.z, rgb[0], rgb[1], rgb[2]);
        radius_i = (int)s.radius;
        tiles = (uint32_t)((x1 - x0) * (y1 - y0));
      }
    }
    if (tiles == 0) x0 = y0 = x1 = y1 = 0;
    g.radii[idx] = radius_i;
    if (a.radii_out) a.radii_out[idx] = radius_i;
    g.rect[idx] = pack_rect(x0, y0, x1, y1);
    tmask = tiles >= 32 ? 0xffffffffu : ((1u << tiles) - 1u);  // no exact tile culling: the whole rect
    g.tile_mask[idx] = tmask;
  }
  // num_rendered = sum of the rect areas: one atomic per warp
  const unsigned wsum = __reduce_add_sync(0xffffffffu, tiles);
  if ((threadIdx.x & 31) == 0 && wsum) atomicAdd(&im.hdr->num_rect, (unsigned long long)wsum);
  // sub-binned tile histogram
  const int T = a.gx * a.gy, warp_base = idx - (int)(threadIdx.x & 31);
  for_each_tile(x0, y0, x1, y1, tmask, a.gx, [&](int tile, unsigned src) {
    atomicAdd(&im.tile_count[subbin_of(warp_base + (int)src) * T + tile], 1u);
  });
}

// ---- compositing forward: one CTA per 16x16 tile, records staged in batches of 256 ---------------------------------
__global__ void __launch_bounds__(CB) k_surfel_render_fwd(int W, int H, int gx, SurfImage si, BinView b, SurfGeom g,
                                                          const float* __restrict__ bg, float* __restrict__ out_color,
                                                          float* __restrict__ out_map) {
  __shared__ float4 sA[CB][REC_A];
  __shared__ float4 sB[CB][REC_B];
  const int tile = blockIdx.x, t = threadIdx.x;
  const int x = (tile % gx) * TILE_X + (t & 15), y = (tile / gx) * TILE_Y + (t >> 4);
  const bool inside = x < W && y < H;
  const uint2 range = si.im.tile_range[tile];
  const float fx = (float)x, fy = (float)y;
  float T = 1.f, C[3] = {0.f, 0.f, 0.f}, D = 0.f, N[3] = {0.f, 0.f, 0.f}, M1 = 0.f, M2 = 0.f, dist = 0.f;
  float med_z = 0.f, med_w = 0.f, med_id = 0.f;
  uint32_t contrib = 0, last = 0, med_c = 0;
  bool done = !inside;
  for (uint32_t base = range.x; base < range.y; base += CB) {
    if (__syncthreads_count(done) == CB) break;  // also: every thread is done with the previous batch
    if (base + t < range.y) {
      const uint32_t gid = b.point_list[base + t];
#pragma unroll
      for (int k = 0; k < REC_A; k++) sA[t][k] = g.recA[(size_t)gid * REC_A + k];
#pragma unroll
      for (int k = 0; k < REC_B; k++) sB[t][k] = g.recB[(size_t)gid * REC_B + k];
    }
    __syncthreads();
    const int n = (int)min((uint32_t)CB, range.y - base);
    for (int j = 0; !done && j < n; j++) {
      contrib++;
      const float4 a0 = sA[j][0], a1 = sA[j][1], a2 = sA[j][2], b0 = sB[j][0], b1 = sB[j][1];
      Pair q;
      if (!eval_pair(fx, fy, a0.x, a0.y, {a2.x, a2.y, a2.z}, {a2.w, b0.x, b0.y}, {a0.z, a0.w, a1.x}, q)) continue;
      const float alpha = fminf(0.99f, a1.y * pair_gauss(q));
      if (alpha < 1.0f / 255.0f) continue;
      const float test_T = T * (1.f - alpha);
      if (test_T < 0.0001f) { done = true; break; }
      const float w = alpha * T;
      C[0] += b1.y * w; C[1] += b1.z * w; C[2] += b1.w * w;
      D += q.z * w;
      N[0] += b0.z * w; N[1] += b0.w * w; N[2] += b1.x * w;
      const float m = dist_m(q.z), A = 1.f - T;
      dist += (m * m * A + M2 - 2.f * m * M1) * w;
      M1 += m * w;
      M2 += m * m * w;
      if (T > 0.5f) { med_z = q.z; med_w = w; med_id = (float)__float_as_int(a1.w); med_c = contrib; }
      T = test_T;
      last = contrib;
    }
  }
  if (!inside) return;
  const size_t HW = (size_t)W * H, pix = (size_t)y * W + x;
#pragma unroll
  for (int c = 0; c < 3; c++) out_color[c * HW + pix] = C[c] + T * bg[c];
  const float maps[9] = {D, 1.f - T, N[0], N[1], N[2], med_z, dist, med_w, med_id};
#pragma unroll
  for (int c = 0; c < 9; c++) out_map[c * HW + pix] = maps[c];
  si.im.final_T[pix] = T;
  si.im.n_contrib[pix] = last;
  si.M1[pix] = M1;
  si.M2[pix] = M2;
  si.med_c[pix] = med_c;
}

// ---- compositing backward: back to front over each tile's list -----------------------------------------------------
// Per pair: dL/dalpha from suffix sums (the 3DGS recursion, one per blended quantity; the distortion's per-splat term
// e_i = m_i^2 (1-T) - 2 m_i M1 + M2 only needs the pixel's final sums), then dL/drho and dL/dz through the branch the
// forward took.  The 18 per-Gaussian sums are reduced over the warp (every lane walks the same list entry) and added to
// the accumulator with one red.global per sum.
__global__ void __launch_bounds__(CB) k_surfel_render_bwd(int W, int H, int gx, SurfImage si, BinView b, SurfGeom g,
                                                          const float* __restrict__ bg, const float* __restrict__ dL_dpix,
                                                          const float* __restrict__ dL_dmap) {
  __shared__ float4 sA[CB][REC_A];
  __shared__ float4 sB[CB][REC_B];
  __shared__ unsigned s_maxc;
  const int tile = blockIdx.x, t = threadIdx.x, lane = t & 31;
  const int x = (tile % gx) * TILE_X + (t & 15), y = (tile / gx) * TILE_Y + (t >> 4);
  const bool inside = x < W && y < H;
  const uint2 range = si.im.tile_range[tile];
  const float fx = (float)x, fy = (float)y;
  const size_t HW = (size_t)W * H, pix = inside ? (size_t)y * W + x : 0;
  const float Tf = inside ? si.im.final_T[pix] : 1.f;
  const uint32_t last = inside ? si.im.n_contrib[pix] : 0u, medc = inside ? si.med_c[pix] : 0u;
  const float M1f = inside ? si.M1[pix] : 0.f, M2f = inside ? si.M2[pix] : 0.f, Af = 1.f - Tf;
  float gC[3] = {0.f, 0.f, 0.f}, gN[3] = {0.f, 0.f, 0.f}, gD = 0.f, gA = 0.f, gMed = 0.f, gDist = 0.f;
  if (inside) {
#pragma unroll
    for (int c = 0; c < 3; c++) { gC[c] = dL_dpix[c * HW + pix]; gN[c] = dL_dmap[(2 + c) * HW + pix]; }
    gD = dL_dmap[pix]; gA = dL_dmap[HW + pix]; gMed = dL_dmap[5 * HW + pix]; gDist = dL_dmap[6 * HW + pix];
  }
  if (t == 0) s_maxc = 0;
  __syncthreads();
  if (last) atomicMax(&s_maxc, last);
  __syncthreads();
  const uint32_t end = range.x + s_maxc;
  float T = Tf, SC[3] = {bg[0], bg[1], bg[2]}, SD = 0.f, SN[3] = {0.f, 0.f, 0.f}, SE = 0.f;
  float pa = 0.f, pc[3] = {0.f, 0.f, 0.f}, pz = 0.f, pn[3] = {0.f, 0.f, 0.f}, pe = 0.f;
  for (uint32_t top = end; top > range.x;) {
    const uint32_t lo = top - range.x > (uint32_t)CB ? top - CB : range.x;
    __syncthreads();  // every thread is done with the previous batch
    if (lo + t < top) {
      const uint32_t gid = b.point_list[lo + t];
#pragma unroll
      for (int k = 0; k < REC_A; k++) sA[t][k] = g.recA[(size_t)gid * REC_A + k];
#pragma unroll
      for (int k = 0; k < REC_B; k++) sB[t][k] = g.recB[(size_t)gid * REC_B + k];
    }
    __syncthreads();
    for (int j = (int)(top - lo) - 1; j >= 0; j--) {
      const uint32_t rel = lo + j - range.x;  // position in the tile's list
      float acc[18];
#pragma unroll
      for (int k = 0; k < 18; k++) acc[k] = 0.f;
      bool hit = false;
      const float4 a0 = sA[j][0], a1 = sA[j][1], a2 = sA[j][2], b0 = sB[j][0], b1 = sB[j][1];
      if (rel < last) {
        const F3 Tu = {a2.x, a2.y, a2.z}, Tv = {a2.w, b0.x, b0.y}, Tw = {a0.z, a0.w, a1.x};
        Pair q;
        if (eval_pair(fx, fy, a0.x, a0.y, Tu, Tv, Tw, q)) {
          const float G = pair_gauss(q), o = a1.y, oG = o * G;
          const float alpha = fminf(0.99f, oG);
          if (!(alpha < 1.0f / 255.0f)) {
            hit = true;
            T = T / (1.f - alpha);
            const float w = alpha * T;
            const float rgb[3] = {b1.y, b1.z, b1.w}, n[3] = {b0.z, b0.w, b1.x};
            const float m = dist_m(q.z), e = m * m * Af - 2.f * m * M1f + M2f;
            float dLda = 0.f;
#pragma unroll
            for (int c = 0; c < 3; c++) {
              SC[c] = pa * pc[c] + (1.f - pa) * SC[c];
              SN[c] = pa * pn[c] + (1.f - pa) * SN[c];
              dLda += gC[c] * (rgb[c] - SC[c]) + gN[c] * (n[c] - SN[c]);
              acc[15 + c] = w * gC[c];
              acc[11 + c] = w * gN[c];
            }
            SD = pa * pz + (1.f - pa) * SD;
            SE = pa * pe + (1.f - pa) * SE;
            dLda += gD * (q.z - SD) + gDist * (e - SE);
            dLda = T * dLda + gA * Tf / (1.f - alpha);
            pa = alpha; pz = q.z; pe = e;
#pragma unroll
            for (int c = 0; c < 3; c++) { pc[c] = rgb[c]; pn[c] = n[c]; }
            float gz = w * gD + gDist * 2.f * w * (m * Af - M1f) * dist_dm(q.z);
            if (rel + 1 == medc) gz += gMed;
            float dLdrho = 0.f;
            if (oG <= 0.99f) {  // the 0.99 clamp passes no gradient
              acc[14] = dLda * G;
              dLdrho = -0.5f * G * o * dLda;
            }
            if (q.rho3 <= q.rho2) {
              const float gsx = dLdrho * 2.f * q.sx + gz * Tw.x, gsy = dLdrho * 2.f * q.sy + gz * Tw.y;
              const F3 gp = {gsx / q.p.z, gsy / q.p.z, -(gsx * q.sx + gsy * q.sy) / q.p.z};
              const F3 gk = cross3(q.l, gp), gl = cross3(gp, q.k);
              acc[2] = -gk.x; acc[3] = -gk.y; acc[4] = -gk.z;
              acc[5] = -gl.x; acc[6] = -gl.y; acc[7] = -gl.z;
              acc[8] = gz * q.sx + fx * gk.x + fy * gl.x;
              acc[9] = gz * q.sy + fx * gk.y + fy * gl.y;
              acc[10] = gz + fx * gk.z + fy * gl.z;
            } else {
              acc[0] = dLdrho * 4.f * (a0.x - fx);
              acc[1] = dLdrho * 4.f * (a0.y - fy);
              acc[10] = gz;
            }
          }
        }
      }
      if (__any_sync(0xffffffffu, hit)) {
#pragma unroll
        for (int k = 0; k < 18; k++) {
          float v = acc[k];
#pragma unroll
          for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
          acc[k] = v;
        }
        if (lane == 0) {
          const int gid = __float_as_int(a1.w);
          float* dst = g.grad + (size_t)gid * SURF_GRAD;
#pragma unroll
          for (int k = 0; k < 18; k++)
            if (acc[k] != 0.f) atomicAdd(dst + k, acc[k]);
        }
      }
    }
    top = lo;
  }
}

// ---- projection backward: one thread per Gaussian, from the accumulator to the input gradients ---------------------
struct SurfBwdArgs {
  int P, D, M, W, H;
  const float *means3D, *shs, *scales, *rotations, *view, *proj, *campos;
  float mod;
  float *dL_dmean2D, *dL_dopacity, *dL_dcolor, *dL_dmean3D, *dL_dsh, *dL_dscale, *dL_drot;
};
__global__ void __launch_bounds__(SURF_THREADS) k_surfel_project_bwd(SurfBwdArgs a, SurfGeom g) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= a.P) return;
  float gm3[3] = {0.f, 0.f, 0.f}, gm2[2] = {0.f, 0.f}, gs[2] = {0.f, 0.f}, gq[4] = {0.f, 0.f, 0.f, 0.f}, go = 0.f;
  float grgb[3] = {0.f, 0.f, 0.f};
  SurfProj s;
  const bool live = g.radii[idx] > 0 && surfel_project(idx, a.means3D, a.scales, a.rotations, a.mod, a.view, a.proj, a.W, a.H, s);
  float w[16] = {0.f};
  F3 gw[16];
  int nco = 0;
  float graw[3] = {0.f, 0.f, 0.f};
  if (live) {
    const float* acc = g.grad + (size_t)idx * SURF_GRAD;
    const float gmx = acc[0], gmy = acc[1];
    F3 gTu = {acc[2], acc[3], acc[4]}, gTv = {acc[5], acc[6], acc[7]}, gTw = {acc[8], acc[9], acc[10]};
    const F3 gnv = {acc[11], acc[12], acc[13]};
    go = acc[14];
    grgb[0] = acc[15]; grgb[1] = acc[16]; grgb[2] = acc[17];
    // screen-space translation statistic (Tu += dx Tw, Tv += dy Tw, mean2D += d), in NDC units
    gm2[0] = (dot3(gTu, s.Tw) + gmx) * 0.5f * a.W;
    gm2[1] = (dot3(gTv, s.Tw) + gmy) * 0.5f * a.H;
    // mean2D = (Tu'Q Tw, Tv'Q Tw) / d, d = Tw'Q Tw
    const F3 QTw = {9.f * s.Tw.x, 9.f * s.Tw.y, -s.Tw.z}, QTu = {9.f * s.Tu.x, 9.f * s.Tu.y, -s.Tu.z},
             QTv = {9.f * s.Tv.x, 9.f * s.Tv.y, -s.Tv.z};
    const float id = 1.f / s.d, cm = 2.f * (gmx * s.mx + gmy * s.my) * id;
    gTu = {gTu.x + gmx * QTw.x * id, gTu.y + gmx * QTw.y * id, gTu.z + gmx * QTw.z * id};
    gTv = {gTv.x + gmy * QTw.x * id, gTv.y + gmy * QTw.y * id, gTv.z + gmy * QTw.z * id};
    gTw = {gTw.x + (gmx * QTu.x + gmy * QTv.x) * id - cm * QTw.x, gTw.y + (gmx * QTu.y + gmy * QTv.y) * id - cm * QTw.y,
           gTw.z + (gmx * QTu.z + gmy * QTv.z) * id - cm * QTw.z};
    // T rows -> clip coordinates of (t_u, t_v, centre): columns 0, 1, 2 of Tu / Tv / Tw
    const float aW = 0.5f * a.W, bW = 0.5f * (a.W - 1), aH = 0.5f * a.H, bH = 0.5f * (a.H - 1);
    const float gTuA[3] = {gTu.x, gTu.y, gTu.z}, gTvA[3] = {gTv.x, gTv.y, gTv.z}, gTwA[3] = {gTw.x, gTw.y, gTw.z};
    float gvec[3][3];  // d L / d (t_u, t_v, p) in world space
#pragma unroll
    for (int j = 0; j < 3; j++) {
      const float gc[4] = {aW * gTuA[j], aH * gTvA[j], 0.f, bW * gTuA[j] + bH * gTvA[j] + gTwA[j]};
#pragma unroll
      for (int r = 0; r < 3; r++)
        gvec[j][r] = gc[0] * a.proj[4 * r] + gc[1] * a.proj[4 * r + 1] + gc[3] * a.proj[4 * r + 3];
    }
    // normal: n_view = sign * (n @ view[:3,:3])
    float gnw[3];
#pragma unroll
    for (int r = 0; r < 3; r++) gnw[r] = s.sign * (gnv.x * a.view[4 * r] + gnv.y * a.view[4 * r + 1] + gnv.z * a.view[4 * r + 2]);
    gs[0] = (gvec[0][0] * s.R[0][0] + gvec[0][1] * s.R[1][0] + gvec[0][2] * s.R[2][0]) * a.mod;
    gs[1] = (gvec[1][0] * s.R[0][1] + gvec[1][1] * s.R[1][1] + gvec[1][2] * s.R[2][1]) * a.mod;
    float gR[3][3];
#pragma unroll
    for (int r = 0; r < 3; r++) { gR[r][0] = gvec[0][r] * s.su; gR[r][1] = gvec[1][r] * s.sv; gR[r][2] = gnw[r]; }
    const float4 q = reinterpret_cast<const float4*>(a.rotations)[idx];
    const float qw = q.x, qx = q.y, qy = q.z, qz = q.w;
    gq[0] = 2.f * (-qz * gR[0][1] + qy * gR[0][2] + qz * gR[1][0] - qx * gR[1][2] - qy * gR[2][0] + qx * gR[2][1]);
    gq[1] = 2.f * (qy * gR[0][1] + qz * gR[0][2] + qy * gR[1][0] - 2.f * qx * gR[1][1] - qw * gR[1][2] + qz * gR[2][0] +
                   qw * gR[2][1] - 2.f * qx * gR[2][2]);
    gq[2] = 2.f * (-2.f * qy * gR[0][0] + qx * gR[0][1] + qw * gR[0][2] + qx * gR[1][0] + qz * gR[1][2] - qw * gR[2][0] +
                   qz * gR[2][1] - 2.f * qy * gR[2][2]);
    gq[3] = 2.f * (-2.f * qz * gR[0][0] - qw * gR[0][1] + qx * gR[0][2] + qw * gR[1][0] - 2.f * qz * gR[1][1] +
                   qy * gR[1][2] + qx * gR[2][0] + qy * gR[2][1]);
    gm3[0] = gvec[2][0]; gm3[1] = gvec[2][1]; gm3[2] = gvec[2][2];
    if (a.shs) {
      float len;
      const F3 dir = view_dir(idx, a.means3D, a.campos, len);
      nco = sh_basis(a.D, dir, w, gw);
      const unsigned char cl = g.clamped[idx];
#pragma unroll
      for (int c = 0; c < 3; c++) graw[c] = (cl >> c) & 1 ? 0.f : grgb[c];
      const float* sh = a.shs + (size_t)idx * a.M * 3;
      F3 gdir = {0.f, 0.f, 0.f};
      for (int k = 1; k < nco; k++) {
        const float f = graw[0] * sh[3 * k] + graw[1] * sh[3 * k + 1] + graw[2] * sh[3 * k + 2];
        gdir = {gdir.x + f * gw[k].x, gdir.y + f * gw[k].y, gdir.z + f * gw[k].z};
      }
      const float dd = dot3(dir, gdir);
      gm3[0] += (gdir.x - dir.x * dd) / len;
      gm3[1] += (gdir.y - dir.y * dd) / len;
      gm3[2] += (gdir.z - dir.z * dd) / len;
    }
  }
  // every output element is written (no pre-zeroing by the caller)
#pragma unroll
  for (int c = 0; c < 3; c++) {
    a.dL_dmean3D[3 * idx + c] = gm3[c];
    a.dL_dcolor[3 * idx + c] = grgb[c];
  }
  a.dL_dmean2D[3 * idx] = gm2[0];
  a.dL_dmean2D[3 * idx + 1] = gm2[1];
  a.dL_dmean2D[3 * idx + 2] = 0.f;
  a.dL_dopacity[idx] = go;
  a.dL_dscale[2 * idx] = gs[0];
  a.dL_dscale[2 * idx + 1] = gs[1];
  reinterpret_cast<float4*>(a.dL_drot)[idx] = make_float4(gq[0], gq[1], gq[2], gq[3]);
  if (a.dL_dsh) {
    float* o = a.dL_dsh + (size_t)idx * a.M * 3;
    for (int k = 0; k < a.M; k++)
#pragma unroll
      for (int c = 0; c < 3; c++) o[3 * k + c] = k < nco ? w[k] * graw[c] : 0.f;
  }
}

const char* surfel_args_error(int P, int D, int M, int W, int H, const float* means3D, const float* shs,
                              const float* colors, const float* scales, const float* rotations, const float* view,
                              const float* proj, const float* campos, const float* bg) {
  if (P < 0) return "P must be >= 0";
  if (W <= 0 || H <= 0) return "width and height must be positive";
  if ((W + TILE_X - 1) / TILE_X > 65535 || (H + TILE_Y - 1) / TILE_Y > 65535) return "image too large";
  if (!bg || !view || !proj) return "background, viewmatrix and projmatrix are required";
  if (P > 0 && (!means3D || !scales || !rotations)) return "means3D, scales and rotations are required";
  if (P > 0 && (shs == nullptr) == (colors == nullptr)) return "need exactly one of shs and colors_precomp";
  if (shs && (D < 0 || D > 3 || (D + 1) * (D + 1) > M)) return "sh degree / coefficient count mismatch (D in 0..3, (D+1)^2 <= M)";
  if (shs && !campos) return "campos is required with shs";
  if (misaligned16(rotations)) return "rotations must be 16-byte aligned";
  return nullptr;
}

}  // namespace
}  // namespace gsr

using namespace gsr;

extern "C" {

size_t gsr_surfel_geometry_bytes(int P) { return sgeom_bytes(P < 0 ? 0 : P); }
size_t gsr_surfel_image_bytes(int width, int height) { return simage_bytes(width < 0 ? 0 : width, height < 0 ? 0 : height); }

int64_t gsr_surfel_forward(gsr_alloc_fn geometry_alloc, void* geometry_user, gsr_alloc_fn binning_alloc,
                           void* binning_user, gsr_alloc_fn image_alloc, void* image_user, int P, int D, int M,
                           const float* background, int width, int height, const float* means3D, const float* shs,
                           const float* colors_precomp, const float* opacities, const float* scales,
                           float scale_modifier, const float* rotations, const float* viewmatrix,
                           const float* projmatrix, const float* cam_pos, int prefiltered, float* out_color,
                           float* out_allmap, int* radii, int debug, void* stream) {
  (void)prefiltered;
  const char* fn = "gsr_surfel_forward";
  if (const char* e = surfel_args_error(P, D, M, width, height, means3D, shs, colors_precomp, scales, rotations,
                                        viewmatrix, projmatrix, cam_pos, background))
    return fail(fn, e);
  if (!geometry_alloc || !binning_alloc || !image_alloc || !out_color || !out_allmap || (P > 0 && !opacities))
    return fail(fn, "allocators, opacities, out_color and out_allmap are required");
  const cudaStream_t st = (cudaStream_t)stream;
  const int W = width, H = height, gx = (W + TILE_X - 1) / TILE_X, gy = (H + TILE_Y - 1) / TILE_Y, T = gx * gy;
  char* gbuf = geometry_alloc(geometry_user, sgeom_bytes(P));
  char* ibuf = image_alloc(image_user, simage_bytes(W, H));
  if (!gbuf || !ibuf) return fail(fn, "scratch allocation failed");
  const SurfGeom g = carve_sgeom(aligned_base(gbuf), P);
  const SurfImage si = carve_simage(aligned_base(ibuf), W, H);
  if (!check(cudaMemsetAsync(si.im.tile_count, 0, sizeof(uint32_t) * T * SUBBINS, st), "memset tile_count")) return -1;
  launch_init_header(si.im.hdr, ~0ull, st);
  if (P > 0) {
    SurfArgs a{P, D, M, W, H, gx, gy, means3D, shs, colors_precomp, opacities, scales, rotations, viewmatrix,
               projmatrix, cam_pos, scale_modifier, radii};
    k_surfel_project<<<(P + SURF_THREADS - 1) / SURF_THREADS, SURF_THREADS, 0, st>>>(a, g, si.im);
  }
  if (!stage_ok(debug, st, "surfel_project")) return -1;
  launch_tile_scan(si.im, T, st);
  if (!stage_ok(debug, st, "tile_scan")) return -1;
  // the one blocking read: the instance count sizes the binning buffer
  unsigned long long counts[2] = {0, 0};  // {binned, rect-sum}: adjacent header fields (equal here: no tile culling)
  cudaError_t e = cudaMemcpyAsync(counts, &si.im.hdr->num_rendered, sizeof(counts), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (!check(e, "read R")) return -1;
  const long long binned = (long long)counts[0];
  char* bbuf = binning_alloc(binning_user, binning_bytes(binned));
  if (!bbuf) return fail(fn, "binning allocation failed");
  const BinView b = carve_binning(aligned_base(bbuf), binned);
  if (binned > 0) {
    launch_scatter(P, gx, T, binning_view(g), si.im, b, st);
    if (!stage_ok(debug, st, "scatter")) return -1;
    launch_tile_sort(T, binning_view(g), si.im, b, st);
    if (!stage_ok(debug, st, "tile_sort")) return -1;
  }
  k_surfel_render_fwd<<<T, CB, 0, st>>>(W, H, gx, si, b, g, background, out_color, out_allmap);
  if (!stage_ok(debug, st, "surfel_render_fwd")) return -1;
  return (int64_t)counts[1];
}

int gsr_surfel_backward(int P, int D, int M, int64_t R, const float* background, int width, int height,
                        const float* means3D, const float* shs, const float* scales, float scale_modifier,
                        const float* rotations, const float* viewmatrix, const float* projmatrix, const float* campos,
                        char* geom_buffer, char* binning_buffer, char* image_buffer, const float* dL_dpix,
                        const float* dL_dallmap, float* dL_dmean2D, float* dL_dopacity, float* dL_dcolor,
                        float* dL_dmean3D, float* dL_dsh, float* dL_dscale, float* dL_drot, int debug, void* stream) {
  // shs == NULL: colours were precomputed (the argument check wants exactly one of shs / colors_precomp)
  static const float kAny = 0.f;
  const char* fn = "gsr_surfel_backward";
  if (const char* e = surfel_args_error(P, D, M, width, height, means3D, shs, shs ? nullptr : &kAny, scales,
                                        rotations, viewmatrix, projmatrix, campos, background))
    return fail(fn, e);
  if (P == 0) return 0;
  if (!geom_buffer || !image_buffer || (R > 0 && !binning_buffer) || R < 0) return fail(fn, "missing state buffers");
  if (!dL_dpix || !dL_dallmap || !dL_dmean2D || !dL_dopacity || !dL_dcolor || !dL_dmean3D || !dL_dscale || !dL_drot ||
      (shs && !dL_dsh))
    return fail(fn, "upstream gradients and every output gradient (dL_dsh with shs) are required");
  if (misaligned16(dL_drot)) return fail(fn, "dL_drot must be 16-byte aligned");
  const cudaStream_t st = (cudaStream_t)stream;
  const int W = width, H = height, gx = (W + TILE_X - 1) / TILE_X, gy = (H + TILE_Y - 1) / TILE_Y;
  const SurfGeom g = carve_sgeom(aligned_base(geom_buffer), P);
  if (!check(cudaMemsetAsync(g.grad, 0, sizeof(float) * SURF_GRAD * (size_t)P, st), "memset grad")) return -1;
  if (R > 0) {
    const SurfImage si = carve_simage(aligned_base(image_buffer), W, H);
    const BinView b = carve_binning(aligned_base(binning_buffer), R);
    k_surfel_render_bwd<<<gx * gy, CB, 0, st>>>(W, H, gx, si, b, g, background, dL_dpix, dL_dallmap);
    if (!stage_ok(debug, st, "surfel_render_bwd")) return -1;
  }
  SurfBwdArgs a{P, D, M, W, H, means3D, shs, scales, rotations, viewmatrix, projmatrix, campos, scale_modifier,
                dL_dmean2D, dL_dopacity, dL_dcolor, dL_dmean3D, dL_dsh, dL_dscale, dL_drot};
  k_surfel_project_bwd<<<(P + SURF_THREADS - 1) / SURF_THREADS, SURF_THREADS, 0, st>>>(a, g);
  return stage_ok(debug, st, "surfel_project_bwd") ? 0 : -1;
}

}  // extern "C"
