// Internal declarations of libgsr_b200: buffer layouts, launch wrappers, device helpers.
// H100 (sm_90a) only.  Not part of the public ABI (that is include/gsr.h).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>

namespace gsr {

constexpr int TILE_X = 16;  // observable behaviour of the reference (config.h:16-17; SURVEY.md §8b)
constexpr int TILE_Y = 16;
constexpr int TILE_PIX = TILE_X * TILE_Y;
// Level-1 binning counters are split into SUBBINS independent counters per tile (chosen by the Gaussian
// index) laid out sub-bin-major, so that the returning atomics of the scatter pass do not serialise on one
// L2 address per hot tile.  A tile's instances are the concatenation of its sub-bin segments.
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
  uint32_t* tile_cursor;  // [SUBBINS][T] write cursors of the scatter pass
  uint32_t* tile_maxc;    // [T] max n_contrib over the tile's pixels (bounds the backward traversal)
  uint32_t* big_tiles;    // [T] compact list of crowded tiles (hdr->num_big entries), built by the scan
  uint32_t* tile_order;   // [T] tiles by decreasing instance count (64 size classes): CTA i of the per-tile kernels
                          //     takes tile_order[i], so the long tiles start first and the short ones fill the tail
};
struct BinView {               // point_list comes FIRST: its address does not depend on the capacity (backward, export)
  uint32_t* point_list;       // [cap] Gaussian index per sorted tile instance (== BinningState::point_list)
  unsigned long long* ents;   // [cap] (depth bits << 32 | gaussian index), grouped by tile (level-1 output)
  unsigned long long* ents2;  // [cap] scratch of the level-2 sort for tiles that exceed shared memory
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
void launch_preprocess_fwd(const FwdArgs& a, GeomView g, ImageView im, cudaStream_t st);
void launch_tile_scan(ImageView im, int T, cudaStream_t st);
int set_tile_order(int mode);  // gsr_set_tile_order
void launch_scatter(int P, int gx, int T, GeomView g, ImageView im, BinView b, cudaStream_t st);
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
void launch_mark_visible(int P, const float* means3D, const float* view, const float* proj,
                         unsigned char* present, cudaStream_t st);
void launch_depth2normal(const float* depth, int W, int H, float fx, float fy, float cx, float cy, float dmin,
                         float dmax, const float* rot, float* out, cudaStream_t st);
void launch_depth2point(const float* depth, int W, int H, float fx, float fy, float cx, float cy, const float* c2w,
                        float* out, cudaStream_t st);
void launch_debug_export(int P, int W, int H, long long R, GeomView g, BinView b, ImageView im,
                         uint32_t* point_list, uint32_t* ranges, uint32_t* n_contrib, float* final_T,
                         float* means2D, float* conic_opacity, float* depths, float* rgb, float* cov3D,
                         uint32_t* tiles_touched, unsigned char* clamped, cudaStream_t st);

// ---- small device helpers shared by the kernels ----
// model activations of gaustudio's VanillaPointCloud (models/vanilla_sg.py:29-35, models/utils.py:6-32)
__device__ __forceinline__ float act_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ float4 act_normalize(float4 q, float* inv_norm = nullptr) {
  const float n = fmaxf(sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w), 1e-12f);  // F.normalize eps
  if (inv_norm) *inv_norm = 1.0f / n;
  return make_float4(q.x / n, q.y / n, q.z / n, q.w / n);
}
__device__ __forceinline__ int subbin_of(int gaussian_idx) { return gaussian_idx & (SUBBINS - 1); }
__device__ __forceinline__ uint2 pack_rect(int xmin, int ymin, int xmax, int ymax) {
  return make_uint2((unsigned)xmin | ((unsigned)xmax << 16), (unsigned)ymin | ((unsigned)ymax << 16));
}
__device__ __forceinline__ void unpack_rect(uint2 r, int& xmin, int& ymin, int& xmax, int& ymax) {
  xmin = r.x & 0xffff; xmax = r.x >> 16; ymin = r.y & 0xffff; ymax = r.y >> 16;
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

// gsr_extract.cu -- the extraction post-pass (gaustudio/scripts/extract_pcd.py)
struct SpaceKernel { float w[225]; };  // (2r+1)^2 spatial weights of the bilateral filter, 0 outside the disc
void launch_masked_bilateral(const float* depth, const unsigned char* mask, int W, int H, int r, float gauss_color,
                             const SpaceKernel& sk, float* out_depth, unsigned char* out_mask, unsigned* scratch,
                             cudaStream_t st);
void launch_extract_normals(const float* depth, const unsigned char* fg, const float* opacity, const float* median_depth,
                            int W, int H, float fx, float fy, float cx, float cy, const float* rot, float depth_limit,
                            float opacity_min, float* cam_normals, float* neg_world, unsigned char* valid,
                            cudaStream_t st);
void launch_fusion_pass(long long n, const long long* ids, const float* normals, const float* conf, int P,
                        const float* xyz, float tx, float ty, float tz, const float* mean, float thresh,
                        float* sum_normals, float* sum_weights, unsigned char* touched, cudaStream_t st);
void launch_fusion_mean(int P, const float* sum_normals, const float* sum_weights, float* mean, cudaStream_t st);
int launch_knn_grid(int n, int k, const float* pts, const int* cell_start, const float* grid, int* out_index,
                    float* out_dist, cudaStream_t st);  // -1: unsupported k (1, 4, 8, 10, 16)
}  // namespace gsr
struct gsr_adam_group;
namespace gsr {
int launch_adam(int n_groups, const gsr_adam_group* groups, double beta1, double beta2, double eps, long long step,
                int decoupled, float grad_scale, int zero_grad, cudaStream_t st);

}  // namespace gsr
