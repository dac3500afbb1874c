// Internal declarations of libgsr_b200: buffer layouts, launch wrappers, device helpers.
// H100 (sm_90a) only.  Not part of the public ABI (that is include/gsr.h).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>

#include <string>

namespace gsr {

constexpr int TILE_X = 16;  // observable behaviour of the reference (config.h:16-17; SURVEY.md §8b)
constexpr int TILE_Y = 16;
constexpr int TILE_PIX = TILE_X * TILE_Y;
// The projection's tile histogram is split into SUBBINS independent counters per tile (chosen by the Gaussian
// index) laid out sub-bin-major, so that its atomics do not serialise on one L2 address per hot tile.  The tile
// scan adds them up.
constexpr int SUBBINS = 16;

// ---------------------------------------------------------------------------------------------
// Per-Gaussian projected record ("splat"), 48 B = 3 x float4: what the render kernels stage into shared
// memory for every sorted tile instance (asynchronous 16-byte copies, gsr_render.cu).
//   q0 = { mean2D.x, mean2D.y, conic.A, conic.B }
//   q1 = { conic.C, opacity, view-depth, rgb.r }
//   q2 = { rgb.g, rgb.b, bits(gaussian index), bits(radius) }
// ---------------------------------------------------------------------------------------------
constexpr int SPLAT_F4 = 3;
constexpr int SPLAT_BYTES = 48;
constexpr int GRAD_F = 12;  // per-Gaussian screen-space gradient accumulator (10 used), 48 B

struct ImageHeader {            // first 256 B of the image buffer
  unsigned long long num_rendered;  // binned tile instances = sum of the tile histogram (written by the scan kernel)
  unsigned long long num_rect;      // the reference's num_rendered: sum of the tile-rect areas (projection kernel)
  unsigned long long capacity;      // binning capacity the scatter / sort / render kernels may use
  unsigned int overflow;            // set when num_rendered > capacity (pipelined mode)
  unsigned int num_big;             // tiles with more instances than the small sort kernel holds
  unsigned int ticket[2];           // work counters of the two crowded-tile sort launches (dynamic tile hand-out)
  unsigned int pad[6];
};

struct GeomView {      // carved from the geometry buffer, all 256-B aligned
  float4* splat;       // [P][3]
  uint2* rect;         // [P] packed tile rect: x = xmin | xmax<<16, y = ymin | ymax<<16
  float* cov3D;        // [P][6]
  unsigned char* clamped;  // [P] bit c set <=> channel c was clamped (forward.cu:66-68)
  int* radii;          // [P] (internal copy; the caller's radii array is also written)
  uint32_t* tiles_touched;  // [P] area of the tile rect (the reference's tiles_touched)
  uint32_t* tile_mask;      // [P] rects of <= 32 tiles: bit i set <=> tile i (row-major in the rect) is binned
  float* grad;         // [P][GRAD_F] backward scratch
};
struct ImageView {
  ImageHeader* hdr;
  float* final_T;         // [H*W]
  uint32_t* n_contrib;    // [H*W]
  uint32_t* tile_count;   // [SUBBINS][T] instance histogram (sub-bin major)
  uint2* tile_range;      // [T] [start,end) into the sorted instance list; (0,0) when empty
  uint32_t* tile_cursor;  // [SUBBINS][T] scratch of the scatter: tile cursors, super-tile lists, ticket (BinScratch)
  uint32_t* tile_maxc;    // [T] max n_contrib over the tile's pixels (bounds the backward traversal)
  uint32_t* big_tiles;    // [T] compact list of crowded tiles (hdr->num_big entries), built by the scan
  uint32_t* tile_order;   // [T] tiles by decreasing instance count (64 size classes): CTA i of the per-tile kernels
                          //     takes tile_order[i], so the long tiles start first and the short ones fill the tail
};
struct BinView {               // point_list comes FIRST: its address does not depend on the capacity (backward, export)
  uint32_t* point_list;       // [cap] Gaussian index per sorted tile instance (== BinningState::point_list)
  unsigned long long* ents;   // [cap] (depth bits << 32 | gaussian index), grouped by tile (level-1 output)
  unsigned long long* ents2;  // [cap] super-tile lists of the scatter, then scratch of the level-2 sort for tiles that
                              // exceed shared memory
};

// Launch with an execution priority (cudaLaunchAttributePriority; recorded in the kernel node under graph capture).
// The per-Gaussian and binning kernels are memory- / latency-bound, the compositing kernels issue-bound; when several
// views are in flight on different streams the block scheduler hands out CTAs kernel by kernel in launch order, so
// without a hint a short latency-bound kernel of view B waits behind all 8160 CTAs of view A's compositing kernel and
// the two kinds of work never overlap.  With the high priority its CTAs take the slots that free up first.
// GSR_PRIORITY=0 (read once) launches everything at the default priority.
int high_priority();  // the device's greatest stream priority, or 0 (= default) when disabled (gsr_api.cu)
template <typename... KArgs, typename... Args>
inline cudaError_t launch_high_priority(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                        Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributePriority;
  attr[0].val.priority = high_priority();
  cfg.attrs = attr; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// Per-device facts and one-time kernel attributes of the CURRENT device (cached; gsr_api.cu).
struct DeviceInfo {
  int sm_count = 0;
  mutable bool sort_attr_set = false;
  mutable size_t pre_fwd_smem = 48 * 1024 - 64, pre_bwd_smem = 48 * 1024 - 64;  // dynamic smem opted into so far
};
const DeviceInfo& device_info();

size_t geom_bytes(int P);
size_t image_bytes(int W, int H);
size_t binning_bytes(long long R);
GeomView carve_geom(char* base, int P);
ImageView carve_image(char* base, int W, int H);
BinView carve_binning(char* base, long long cap);

struct FwdArgs {
  int P, D, M, W, H, gx, gy;
  const float *means3D, *shs, *colors_precomp, *opacities, *scales, *rotations, *cov3D_precomp;
  const float *view, *proj, *campos;
  float scale_modifier, tan_fovx, tan_fovy, focal_x, focal_y;
  int prefiltered;
  int* radii_out;
  // fused-activation variant (gsr_forward_fused): scales / rotations / opacities are the model's RAW
  // attributes (log-scale, un-normalised quaternion, opacity logit) and the SH tensor arrives as its two
  // stored pieces f_dc [P,1,3] + f_rest [P,M-1,3]; the kernel applies exp / normalize / sigmoid / cat itself.
  int fused;
  const float *f_dc, *f_rest;
  int sh_bulk;  // f_dc / f_rest are 16-byte aligned: stage each CTA's contiguous SH block with TMA bulk copies
  int sh_rows;  // un-fused [P,16,3] SH tensor, 16-byte aligned: every thread stages its own 192-byte row with TMA
};

// ---- launch wrappers (each enqueues on `st`) ----
// zeroes the header's counters and sets the binning capacity the scatter / sort / render kernels may use
void launch_init_header(ImageHeader* hdr, unsigned long long cap, cudaStream_t st);
void launch_preprocess_fwd(const FwdArgs& a, GeomView g, ImageView im, cudaStream_t st);
void launch_tile_scan(ImageView im, int gx, int gy, cudaStream_t st);
int set_tile_order(int mode);  // gsr_set_tile_order
// two kernels: Gaussians to super-tiles, then to tiles (gsr_binning.cu)
void launch_scatter(int P, int gx, int gy, GeomView g, ImageView im, BinView b, cudaStream_t st);
void launch_tile_sort(int T, GeomView g, ImageView im, BinView b, cudaStream_t st);
// tma: stage the record batches with TMA bulk copies instead of LDGSTS (GSR_FWD_TMA=1)
void launch_render_fwd(int W, int H, int gx, int gy, ImageView im, BinView b, GeomView g, bool tma, float* out_color, float* out_depth, float* out_median, float* out_opacity, cudaStream_t st);
void launch_render_bwd(int W, int H, int gx, int gy, const float* bg, ImageView im, BinView b, GeomView g,
                       const float* dL_dpix, const float* dL_ddepth, const float* dL_dmedian,
                       const float* dL_dopacity, cudaStream_t st);

struct BwdArgs {
  int P, D, M, W, H;
  const float *means3D, *shs, *colors_precomp, *scales, *rotations, *cov3D_precomp;
  const float *view, *proj, *campos;
  float scale_modifier, tan_fovx, tan_fovy, focal_x, focal_y;
  const int* radii;
  float *dL_dmean2D, *dL_dconic, *dL_dopacity, *dL_dcolor, *dL_ddepth, *dL_dmean3D, *dL_dcov3D, *dL_dsh,
      *dL_dscale, *dL_drot;
  // fused-activation variant (gsr_backward_fused): raw inputs, gradients w.r.t. the raw attributes
  int fused;
  const float *f_dc, *f_rest, *opacities_raw;
  float *dL_df_dc, *dL_df_rest;
  int sh_bulk;  // as in FwdArgs; the SH gradient block leaves through a TMA bulk store as well
  int sh_rows;  // as in FwdArgs; gradient rows leave through per-row bulk stores
};
void launch_preprocess_bwd(const BwdArgs& a, GeomView g, cudaStream_t st);
// Mip-Splatting projection (2D Mip filter of width kernel_size instead of the 0.3 dilation); un-fused arguments only
void launch_mip_preprocess_fwd(const FwdArgs& a, GeomView g, ImageView im, float kernel_size, cudaStream_t st);
void launch_mip_preprocess_bwd(const BwdArgs& a, GeomView g, const float* opacities, float kernel_size, cudaStream_t st);
// Scaffold-GS anchor visibility (gsr_scaffold_visible, gsr_scaffold.cu): radii[P] of the Mip projection of width
// kernel_size, un-fused scales [P,3] + rotations [P,4] or cov3D_precomp [P,6]
struct ScaffoldVisArgs {
  int P, W, H;
  const float *means3D, *scales, *rotations, *cov3D_precomp, *view, *proj;
  float scale_modifier, tan_fovx, tan_fovy, kernel_size;
  int* radii;
};
void launch_scaffold_visible(const ScaffoldVisArgs& a, cudaStream_t st);

// ---- small device helpers shared by the kernels ----
// model activations of gaustudio's VanillaPointCloud (models/vanilla_sg.py:29-35, models/utils.py:6-32)
__device__ __forceinline__ float act_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ float4 act_normalize(float4 q, float* inv_norm = nullptr) {
  const float n = fmaxf(sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w), 1e-12f);  // F.normalize eps
  if (inv_norm) *inv_norm = 1.0f / n;
  return make_float4(q.x / n, q.y / n, q.z / n, q.w / n);
}
// sigmoid with each op rounded on its own, as torch's sigmoid kernel rounds them (1 / (1 + exp(-x)))
__device__ __forceinline__ float sigmoid_rn(float x) { return __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-x))); }

// CTA-wide exclusive scan of the count / scan / add kernels of gsr_scaffold.cu and gsr_densify.cu
namespace cta {
constexpr int SCAN_THREADS = 1024;  // items per block of the count; the block totals are scanned by one CTA

// exclusive scan of one value per thread over the CTA (blockDim.x = SCAN_THREADS); returns the CTA total in *total
__device__ __forceinline__ int cta_exclusive_scan(int v, int* total) {
  __shared__ int warp_sum[SCAN_THREADS / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, d);
    if (lane >= d) x += y;
  }
  if (lane == 31) warp_sum[w] = x;
  __syncthreads();
  if (w == 0) {
    int s = warp_sum[lane];
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, s, d);
      if (lane >= d) s += y;
    }
    warp_sum[lane] = s;  // inclusive over warps
  }
  __syncthreads();
  *total = warp_sum[SCAN_THREADS / 32 - 1];
  const int r = x - v + (w > 0 ? warp_sum[w - 1] : 0);
  __syncthreads();  // warp_sum may be reused by the caller's next round
  return r;
}
}  // namespace cta

// CTA-wide sum / max of one double per thread, in a fixed order (warp shuffles, then thread 0 over the warps); the
// result is valid in thread 0.  The per-point reductions of gsr_sap.cu and gsr_clean.cu run RED_CTAS CTAs of
// RED_THREADS threads and add the RED_CTAS partials in one CTA: a fixed grid, so their summation order never changes.
constexpr int RED_CTAS = 256;
constexpr int RED_THREADS = 256;
__device__ __forceinline__ double block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) red[warp] = v;
  __syncthreads();
  v = 0.0;
  if (threadIdx.x == 0)
    for (int k = 0; k < (int)(blockDim.x >> 5); k++) v += red[k];
  __syncthreads();
  return v;
}
__device__ __forceinline__ double block_max(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_down_sync(0xffffffffu, v, o));
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) red[warp] = v;
  __syncthreads();
  v = 0.0;
  if (threadIdx.x == 0)
    for (int k = 0; k < (int)(blockDim.x >> 5); k++) v = fmax(v, red[k]);
  __syncthreads();
  return v;
}

__device__ __forceinline__ int subbin_of(int gaussian_idx) { return gaussian_idx & (SUBBINS - 1); }
__device__ __forceinline__ uint2 pack_rect(int xmin, int ymin, int xmax, int ymax) {
  return make_uint2((unsigned)xmin | ((unsigned)xmax << 16), (unsigned)ymin | ((unsigned)ymax << 16));
}
__device__ __forceinline__ void unpack_rect(uint2 r, int& xmin, int& ymin, int& xmax, int& ymax) {
  xmin = r.x & 0xffff; xmax = r.x >> 16; ymin = r.y & 0xffff; ymax = r.y >> 16;
}

// auxiliary.h:46-56
__device__ __forceinline__ void tile_rect(float px, float py, int max_radius, int gx, int gy, int& x0, int& y0,
                                          int& x1, int& y1) {
  x0 = min(gx, max((int)0, (int)((px - max_radius) / TILE_X)));
  y0 = min(gy, max((int)0, (int)((py - max_radius) / TILE_Y)));
  x1 = min(gx, max((int)0, (int)((px + max_radius + TILE_X - 1) / TILE_X)));
  y1 = min(gy, max((int)0, (int)((py + max_radius + TILE_Y - 1) / TILE_Y)));
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

// ---------------------------------------------------------------------------------------------
// Conservative rectangle test, shared by the binning (16x16 tiles) and the compositing kernels (8x4 blocks).
// Returns false only if alpha = min(0.99, o*exp(power)) < 1/255 for EVERY pixel centre in [rx0,rx1]x[ry0,ry1] (the
// reference skips such pairs, forward.cu:353-355 / backward.cu:535-537).
// With q(d) = A dx^2 + 2B dx dy + C dy^2 = -2*power, alpha >= 1/255 needs q <= tau = 2 ln(255 o) (stored in
// the record by the projection kernel).  q is convex (conic positive definite), so its minimum over the
// rectangle is 0 if the centre is inside, else it lies on an edge facing the centre; each facing edge is a
// 1-D quadratic minimised in closed form.  The edge minimiser uses an approximate reciprocal: an error in the
// minimiser's position only enters q to second order (and not at all when it is clamped to a corner).  The
// margin covers the rounding of the per-pixel evaluation (relative 1e-5 of the largest term magnitude + 1e-3
// absolute); any non-finite / non-PD / extreme input keeps the pair.
// ---------------------------------------------------------------------------------------------
struct CullRec {
  float gx, gy, A, B, C, tau, nBiC, nBiA;  // nBiC = -B / C, nBiA = -B / A
  bool live, odd;                          // live: opacity can reach 1/255 at all; odd: keep unconditionally
};
__device__ __forceinline__ CullRec cull_prep(const float4 q0, const float4 q1, const float tau) {
  CullRec r;
  r.gx = q0.x; r.gy = q0.y; r.A = q0.z; r.B = q0.w; r.C = q1.x; r.tau = tau;
  r.live = !(q1.y < 0.0039f);  // alpha <= o < 1/255 everywhere (exp(power) <= 1)
  r.odd = !(r.A > 1e-30f && r.C > 1e-30f && r.A * r.C - r.B * r.B > 0.f && r.A < 1e30f && r.C < 1e30f);
  float iC, iA;  // A, C in (1e-30, 1e30) whenever the values are used: plain MUFU.RCP is safe
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(iC) : "f"(r.C));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(iA) : "f"(r.A));
  r.nBiC = -r.B * iC;
  r.nBiA = -r.B * iA;
  return r;
}
__device__ __forceinline__ bool may_touch(const CullRec& r, float rx0, float ry0, float rx1, float ry1) {
  if (!r.live) return false;
  const float dxlo = r.gx - rx1, dxhi = r.gx - rx0, dylo = r.gy - ry1, dyhi = r.gy - ry0;
  const bool inx = dxlo <= 0.f && dxhi >= 0.f, iny = dylo <= 0.f && dyhi >= 0.f;
  if ((inx && iny) || r.odd) return true;
  float qmin = 3.0e38f;
  if (!inx) {
    const float dxe = dxlo > 0.f ? dxlo : dxhi;
    const float dys = fminf(fmaxf(r.nBiC * dxe, dylo), dyhi);
    qmin = r.A * dxe * dxe + 2.f * r.B * dxe * dys + r.C * dys * dys;
  }
  if (!iny) {
    const float dye = dylo > 0.f ? dylo : dyhi;
    const float dxs = fminf(fmaxf(r.nBiA * dye, dxlo), dxhi);
    qmin = fminf(qmin, r.A * dxs * dxs + 2.f * r.B * dxs * dye + r.C * dye * dye);
  }
  const float mx = fmaxf(fabsf(dxlo), fabsf(dxhi)), my = fmaxf(fabsf(dylo), fabsf(dyhi));
  const float S = r.A * mx * mx + r.C * my * my + 2.f * fabsf(r.B) * mx * my;
  return !(qmin > r.tau + 1e-5f * S + 1e-3f);
}

// 5-point cross normal of Camera.depth2normal (gaustudio/datasets/__init__.py:106-112,307-380, k = 3), same
// arithmetic order as the reference's torch ops:  u' = (u/(W-1))*(W-1);  X = (u'*z)*Kinv00 + z*Kinv02, ...;
// n = -normalize(cross(top-bottom, left-right)).  False (no output) where the reference writes -1.
__device__ __forceinline__ bool cross_normal(const float* __restrict__ depth, int u, int v, int W, int H, float ifx,
                                             float ify, float ox, float oy, float dmin, float dmax, float& c0,
                                             float& c1, float& c2) {
  if (!(u > 0 && v > 0 && u < W - 1 && v < H - 1)) return false;
  auto point = [&](int uu, int vv, float& x, float& y, float& z) {
    z = depth[(size_t)vv * W + uu];
    const float uz = __fmul_rn(__fmul_rn(__fdiv_rn((float)uu, (float)(W - 1)), (float)(W - 1)), z);
    const float vz = __fmul_rn(__fmul_rn(__fdiv_rn((float)vv, (float)(H - 1)), (float)(H - 1)), z);
    x = __fadd_rn(__fmul_rn(uz, ifx), __fmul_rn(z, ox));
    y = __fadd_rn(__fmul_rn(vz, ify), __fmul_rn(z, oy));
  };
  float cx, cy, cz, tx, ty, tz, bx, by, bz, lx, ly, lz, rx, ry, rz;
  point(u, v, cx, cy, cz); point(u, v - 1, tx, ty, tz); point(u, v + 1, bx, by, bz);
  point(u - 1, v, lx, ly, lz); point(u + 1, v, rx, ry, rz);
  auto ok = [&](float z) { return z > dmin && z < dmax; };
  if (!(ok(cz) && ok(tz) && ok(bz) && ok(lz) && ok(rz))) return false;
  const float ax = tx - bx, ay = ty - by, az = tz - bz, hx = lx - rx, hy = ly - ry, hz = lz - rz;
  c0 = -(__fmul_rn(ay, hz) - __fmul_rn(az, hy));
  c1 = -(__fmul_rn(az, hx) - __fmul_rn(ax, hz));
  c2 = -(__fmul_rn(ax, hy) - __fmul_rn(ay, hx));
  const float len = fmaxf(sqrtf(c0 * c0 + c1 * c1 + c2 * c2), 1e-12f);
  c0 /= len; c1 /= len; c2 /= len;
  return true;
}

// ---- host helpers of the entry points ----
// sets the text gsr_last_error() returns (gsr_api.cu keeps it) to "<entry>: <msg>"; returns -1, the entry's failure
int fail(const char* entry, const std::string& msg);
// what an entry returns after its launches: 0, or -1 with the text "<entry>: <CUDA error text>"
inline int launched(const char* entry) {
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : fail(entry, cudaGetErrorString(e));
}
inline unsigned blocks(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }
bool kernel_size_ok(float k);  // width of a Mip filter: finite and >= 0
// a count the kernels index with int: "<what> must be in 1..2^31-1" otherwise
inline bool count_ok(const char* fn, int64_t n, const char* what) {
  if (n >= 1 && n <= 0x7fffffffLL) return true;
  fail(fn, std::string(what) + " must be in 1..2^31-1");
  return false;
}
// the edge of a dense grid (visual hull, Shape-as-Points)
inline bool res_ok(const char* fn, int res) {
  if (res >= 2 && res <= 512) return true;
  fail(fn, "res must be in 2..512");
  return false;
}
// copies n device words to the host on st and synchronises: 0, or -1 with the entry's error set
template <typename T> inline int read_back(const char* fn, const T* src, T* dst, size_t n, cudaStream_t st) {
  cudaMemcpyAsync(dst, src, n * sizeof(T), cudaMemcpyDeviceToHost, st);
  if (launched(fn)) return -1;
  if (cudaStreamSynchronize(st) != cudaSuccess) { launched(fn); return -1; }
  return 0;
}

inline size_t align256(size_t v) { return (v + 255) / 256 * 256; }
// carves `count` elements from p at its next 256-byte boundary and advances p past them
template <typename T> inline void take(char*& p, T*& out, size_t count) {
  p = reinterpret_cast<char*>(align256(reinterpret_cast<size_t>(p)));
  out = reinterpret_cast<T*>(p);
  p += count * sizeof(T);
}
inline char* aligned_base(char* p) { return reinterpret_cast<char*>(align256(reinterpret_cast<size_t>(p))); }
// Asks `alloc` for one scratch block and carves it: `layout(p)` takes every array from p with take().  The layout runs
// from a null base to size the block (255 bytes more cover an allocation that is not 256-byte aligned), then on the
// allocation.  false: the allocation failed, with the entry's error set.
template <typename Layout>
inline bool carve_scratch(const char* fn, char* (*alloc)(void*, size_t), void* user, Layout layout) {
  char* p = nullptr;
  layout(p);
  char* base = alloc(user, reinterpret_cast<size_t>(p) + 255);
  if (!base) { fail(fn, "scratch allocation failed"); return false; }
  layout(base);
  return true;
}
// the projection kernels move a Gaussian's quaternion (and its gradient, and dL_dconic) as one float4
inline bool misaligned16(const void* p) { return (reinterpret_cast<size_t>(p) & 15) != 0; }

inline bool check(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return true;
  fail(what, cudaGetErrorString(e));
  return false;
}
// CHECK_CUDA of the reference (auxiliary.h:166-173): with debug, synchronise and surface errors per stage
inline bool stage_ok(bool debug, cudaStream_t st, const char* what) {
  if (!check(cudaGetLastError(), what)) return false;
  if (debug && !check(cudaStreamSynchronize(st), what)) return false;
  return true;
}

}  // namespace gsr
