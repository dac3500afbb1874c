// C ABI of the rasterizer (include/gsr.h): buffer carving, stage orchestration, depth maps, state export, and the
// error text of every entry point.  Orchestration restates CudaRasterizer::Rasterizer::{forward,backward}
// ($RAST/cuda_rasterizer/rasterizer_impl.cu:198-343, 347-452) on top of the H100 kernels.
#include "../../include/gsr.h"
#include "gsr_internal.cuh"
#include <cmath>

#include <cstdio>
#include <cstdlib>
#include <atomic>
#include <cstring>
#include <initializer_list>
#include <mutex>
#include <string>
#include <vector>

#include <nvtx3/nvToolsExt.h>  // header-only NVTX v3: ranges cost nothing unless a profiler is attached

namespace gsr {

namespace {
thread_local std::string g_err;
void set_last_error(const char* msg) { g_err = msg; }

// ---- optional per-stage timing (gsr_profile_*) ----
struct ProfRec { int stage; cudaEvent_t a, b; };
bool g_prof_on = false;
std::mutex g_prof_mu;
std::vector<ProfRec> g_prof;
const char* const kStageName[GSR_NUM_STAGES] = {"gsr:preprocess_fwd", "gsr:tile_scan", "gsr:scatter", "gsr:tile_sort",
                                                "gsr:render_fwd", "gsr:render_bwd", "gsr:preprocess_bwd",
                                                "gsr:depth2normal"};
// the stage numbers of gsr_profile_read (gsr.h), in the order of kStageName
enum Stage { kPreprocessFwd, kTileScan, kScatter, kTileSort, kRenderFwd, kRenderBwd, kPreprocessBwd, kDepth2Normal, kNumStages };
static_assert(kNumStages == GSR_NUM_STAGES, "one Stage per profiling stage of gsr.h");
// One per stage launch: an NVTX range (timeline tools) and, when gsr_profile_enable(1), a CUDA-event pair.
struct Prof {
  int stage; cudaStream_t st; cudaEvent_t a = nullptr, b = nullptr;
  Prof(Stage s, cudaStream_t t) : stage(s), st(t) {
    nvtxRangePushA(kStageName[s]);
    if (!g_prof_on) return;
    cudaEventCreate(&a); cudaEventCreate(&b);
    cudaEventRecord(a, st);
  }
  ~Prof() {
    nvtxRangePop();
    if (!a) return;
    cudaEventRecord(b, st);
    std::lock_guard<std::mutex> l(g_prof_mu);
    g_prof.push_back({stage, a, b});
  }
};
}  // namespace

int high_priority() {
  static const int prio = [] {
    const char* e = getenv("GSR_PRIORITY");
    if (e && e[0] == '0') return 0;
    int least = 0, greatest = 0;
    return cudaDeviceGetStreamPriorityRange(&least, &greatest) == cudaSuccess ? greatest : 0;
  }();
  return prio;
}

const DeviceInfo& device_info() {
  static DeviceInfo info[64];
  static std::mutex mu;
  int dev = 0;
  cudaGetDevice(&dev);
  dev = dev < 0 ? 0 : (dev > 63 ? 63 : dev);
  DeviceInfo& d = info[dev];
  if (d.sm_count == 0) {
    std::lock_guard<std::mutex> l(mu);
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;  // H100 SXM
    d.sm_count = n;
  }
  return d;
}

// ---- optional TMA bulk-copy staging of the compositing forward (GSR_FWD_TMA=1, read once per process) ----
namespace {
bool fwd_tma_enabled() {
  static const bool on = [] { const char* e = getenv("GSR_FWD_TMA"); return e && e[0] == '1'; }();
  return on;
}
}  // namespace

GeomView carve_geom(char* base, int P) {
  GeomView g;
  char* p = base;
  take(p, g.splat, (size_t)P * SPLAT_F4);
  take(p, g.rect, (size_t)P);
  take(p, g.cov3D, (size_t)P * 6);
  take(p, g.clamped, (size_t)P);
  take(p, g.radii, (size_t)P);
  take(p, g.tiles_touched, (size_t)P);
  take(p, g.tile_mask, (size_t)P);
  take(p, g.grad, (size_t)P * GRAD_F);
  return g;
}
size_t geom_bytes(int P) {
  GeomView g = carve_geom(nullptr, P);
  return reinterpret_cast<size_t>(g.grad + (size_t)P * GRAD_F) + 512;
}
ImageView carve_image(char* base, int W, int H) {
  ImageView im;
  char* p = base;
  const size_t N = (size_t)W * H;
  const size_t T = (size_t)((W + TILE_X - 1) / TILE_X) * ((H + TILE_Y - 1) / TILE_Y);
  take(p, im.hdr, 1);
  take(p, im.final_T, N);
  take(p, im.n_contrib, N);
  take(p, im.tile_count, T * SUBBINS);
  take(p, im.tile_range, T);
  take(p, im.tile_cursor, T * SUBBINS);
  take(p, im.tile_maxc, T);
  take(p, im.big_tiles, T);
  take(p, im.tile_order, T);
  return im;
}
size_t image_bytes(int W, int H) {
  ImageView im = carve_image(nullptr, W, H);
  const size_t T = (size_t)((W + TILE_X - 1) / TILE_X) * ((H + TILE_Y - 1) / TILE_Y);
  return reinterpret_cast<size_t>(im.tile_order + T) + 512;
}
// The binning arrays are laid out for the instance count rounded up to 1 Mi entries: the buffer size (and with
// it the caller's allocator block) then takes only a few distinct values across views instead of one per view.
static inline long long round_cap(long long n) { return (n + (1ll << 20) - 1) & ~((1ll << 20) - 1); }

BinView carve_binning(char* base, long long cap) {
  BinView b;
  char* p = base;
  cap = round_cap(cap);
  take(p, b.point_list, (size_t)cap + 16);
  take(p, b.ents, (size_t)cap);
  take(p, b.ents2, (size_t)cap);
  return b;
}
size_t binning_bytes(long long R) {
  BinView b = carve_binning(nullptr, R);
  return reinterpret_cast<size_t>(b.ents2 + (size_t)round_cap(R)) + 512;
}

namespace {
__global__ void k_init_header(ImageHeader* h, unsigned long long cap) {
  h->num_rendered = 0;
  h->num_rect = 0;
  h->capacity = cap;
  h->overflow = 0;
  h->num_big = 0;
  h->ticket[0] = 0;
  h->ticket[1] = 0;
}

// ---- speculative exact forward -------------------------------------------------------------------------------------
// Exact mode has to read the binned instance count back before it can size the binning buffer (the reference does the
// same, rasterizer_impl.cu:284), and a blocking read in the MIDDLE of the forward leaves the GPU idle while the host
// wakes up, allocates and launches the second half.  The count of a view is close to the count of the previous view of
// the same (device, P, W, H), so from the second view on the forward sizes the binning buffer for 1.25 x the last count,
// enqueues scatter / sort / compositing right behind the scan and only THEN blocks on the count (an event recorded
// after its copy, not the whole stream).  If the guess was large enough -- the normal case -- nothing else happens: the
// returned num_rendered is exact and the results are the same kernels on the same data.  If it was too small the kernels
// have dropped the overflowing tiles (never an out-of-bounds write); the scan is repeated with the exact capacity and the
// second half runs again.  GSR_SPECULATE=0 / gsr_set_speculation(0): always the plain blocking form.  debug=1: plain form.
std::atomic<int> g_speculate{-1};
std::atomic<long long> g_spec_hits{0}, g_spec_redos{0};
bool speculate_enabled() {
  static const int dflt = [] { const char* e = getenv("GSR_SPECULATE"); return (e && e[0] == '0') ? 0 : 1; }();
  const int v = g_speculate.load(std::memory_order_relaxed);
  return (v >= 0 ? v : dflt) != 0;
}
struct SpecHint { int dev, P, W, H; long long binned; };
std::mutex g_hint_mu;
SpecHint g_hints[16];
int g_hint_n = 0, g_hint_next = 0;
long long hint_get(int dev, int P, int W, int H) {
  std::lock_guard<std::mutex> l(g_hint_mu);
  for (int i = 0; i < g_hint_n; i++)
    if (g_hints[i].dev == dev && g_hints[i].P == P && g_hints[i].W == W && g_hints[i].H == H) return g_hints[i].binned;
  return -1;
}
void hint_put(int dev, int P, int W, int H, long long binned) {
  std::lock_guard<std::mutex> l(g_hint_mu);
  for (int i = 0; i < g_hint_n; i++)
    if (g_hints[i].dev == dev && g_hints[i].P == P && g_hints[i].W == W && g_hints[i].H == H) { g_hints[i].binned = binned; return; }
  const int slot = g_hint_n < 16 ? g_hint_n++ : (g_hint_next++ & 15);
  g_hints[slot] = {dev, P, W, H, binned};
}
// per host thread: 16 pinned bytes for the two counts and the event the host blocks on (re-made when the device changes)
struct SpecHost {
  long long* counts = nullptr;
  cudaEvent_t ev = nullptr;
  int dev = -1;
  bool ready(int d) {
    if (dev == d && counts && ev) return true;
    if (ev) { cudaEventDestroy(ev); ev = nullptr; }
    if (!counts && cudaHostAlloc(reinterpret_cast<void**>(&counts), 16, cudaHostAllocDefault) != cudaSuccess) { counts = nullptr; cudaGetLastError(); return false; }
    if (cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) != cudaSuccess) { ev = nullptr; cudaGetLastError(); return false; }
    dev = d;
    return true;
  }
};
thread_local SpecHost t_spec;
// capacity for a view whose predecessor needed `binned` instances (the carve rounds the arrays up to 1 Mi entries anyway)
inline long long spec_capacity(long long binned) { return binned + binned / 4 + 4096; }

__global__ void k_set_capacity(ImageHeader* h, unsigned long long cap) {
  h->capacity = cap;
  h->overflow = 0;
  h->num_big = 0;
  h->ticket[0] = 0;
  h->ticket[1] = 0;
}

// gaustudio/datasets/__init__.py:106-112,307-380 -- same arithmetic order as the torch ops of the reference:
//   u' = (u/(W-1))*(W-1);  X = (u'*z)*Kinv00 + z*Kinv02, ...;  n = -normalize(cross(top-bottom, left-right))
__global__ void k_depth2normal(const float* __restrict__ depth, int W, int H, float ifx, float ify, float ox, float oy,
                               float dmin, float dmax, const float* __restrict__ rot, float* __restrict__ out) {
  const int u = blockIdx.x * blockDim.x + threadIdx.x, v = blockIdx.y * blockDim.y + threadIdx.y;
  if (u >= W || v >= H) return;
  float* o = out + ((size_t)v * W + u) * 3;
  float n0 = -1.f, n1 = -1.f, n2 = -1.f, c0, c1, c2;
  if (cross_normal(depth, u, v, W, H, ifx, ify, ox, oy, dmin, dmax, c0, c1, c2)) {
    if (rot) {
      n0 = c0 * rot[0] + c1 * rot[3] + c2 * rot[6];
      n1 = c0 * rot[1] + c1 * rot[4] + c2 * rot[7];
      n2 = c0 * rot[2] + c1 * rot[5] + c2 * rot[8];
    } else {
      n0 = c0; n1 = c1; n2 = c2;
    }
  }
  o[0] = n0; o[1] = n1; o[2] = n2;
}

// Camera.depth2point (gaustudio/datasets/__init__.py:106-112,307-339): back-projection of a depth map to camera
// or world coordinates (what extract_mesh.py:95-115 feeds the TSDF fusion with).  c2w: row-major 4x4
// inverse(extrinsics) or NULL.
__global__ void k_depth2point(const float* __restrict__ depth, int W, int H, float ifx, float ify, float ox, float oy,
                              const float* __restrict__ c2w, float* __restrict__ out) {
  const int u = blockIdx.x * blockDim.x + threadIdx.x, v = blockIdx.y * blockDim.y + threadIdx.y;
  if (u >= W || v >= H) return;
  const float z = depth[(size_t)v * W + u];
  const float uz = __fmul_rn(__fmul_rn(__fdiv_rn((float)u, (float)(W - 1)), (float)(W - 1)), z);
  const float vz = __fmul_rn(__fmul_rn(__fdiv_rn((float)v, (float)(H - 1)), (float)(H - 1)), z);
  float x = __fadd_rn(__fmul_rn(uz, ifx), __fmul_rn(z, ox));
  float y = __fadd_rn(__fmul_rn(vz, ify), __fmul_rn(z, oy));
  float zz = z;
  if (c2w) {
    const float wx = c2w[0] * x + c2w[1] * y + c2w[2] * z + c2w[3];
    const float wy = c2w[4] * x + c2w[5] * y + c2w[6] * z + c2w[7];
    const float wz = c2w[8] * x + c2w[9] * y + c2w[10] * z + c2w[11];
    x = wx; y = wy; zz = wz;
  }
  float* o = out + ((size_t)v * W + u) * 3;
  o[0] = x; o[1] = y; o[2] = zz;
}

__global__ void k_export_geom(int P, GeomView g, float* means2D, float* conic_opacity, float* depths, float* rgb,
                              float* cov3D, uint32_t* tiles_touched, unsigned char* clamped) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  const bool vis = g.radii[i] > 0;
  float4 q0 = make_float4(0, 0, 0, 0), q1 = q0, q2 = q0;
  if (vis) { q0 = g.splat[(size_t)i * SPLAT_F4]; q1 = g.splat[(size_t)i * SPLAT_F4 + 1]; q2 = g.splat[(size_t)i * SPLAT_F4 + 2]; }
  if (means2D) { means2D[2 * i] = q0.x; means2D[2 * i + 1] = q0.y; }
  if (conic_opacity) { conic_opacity[4 * i] = q0.z; conic_opacity[4 * i + 1] = q0.w; conic_opacity[4 * i + 2] = q1.x; conic_opacity[4 * i + 3] = q1.y; }
  if (depths) depths[i] = q1.z;
  if (rgb) { rgb[3 * i] = q1.w; rgb[3 * i + 1] = q2.x; rgb[3 * i + 2] = q2.y; }
  if (cov3D) for (int k = 0; k < 6; k++) cov3D[6 * i + k] = vis ? g.cov3D[6 * i + k] : 0.f;
  if (tiles_touched) tiles_touched[i] = g.tiles_touched[i];
  if (clamped) { const unsigned char c = vis ? g.clamped[i] : 0; clamped[3 * i] = c & 1; clamped[3 * i + 1] = (c >> 1) & 1; clamped[3 * i + 2] = (c >> 2) & 1; }
}
__global__ void k_export_list(long long R, const ImageHeader* hdr, BinView b, uint32_t* point_list) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long binned = (long long)min(hdr->num_rendered, hdr->capacity);
  if (i < R) point_list[i] = i < binned ? b.point_list[i] : 0xffffffffu;  // R is the caller's array length
}
__global__ void k_export_image(int N, int T, ImageView im, uint32_t* ranges, uint32_t* n_contrib, float* final_T) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) {
    if (n_contrib) n_contrib[i] = im.n_contrib[i];
    if (final_T) final_T[i] = im.final_T[i];
  }
  if (i < T && ranges) { ranges[2 * i] = im.tile_range[i].x; ranges[2 * i + 1] = im.tile_range[i].y; }
}
}  // namespace

namespace {
// what a forward takes besides the kernels' arguments (FwdArgs)
struct FwdHost {
  gsr_alloc_fn geometry_alloc, binning_alloc, image_alloc;
  void *geometry_user, *binning_user, *image_user;
  float *out_color, *out_depth, *out_median_depth, *out_opacity;
  int debug;
  int64_t r_capacity;  // > 0: pipelined mode
  int64_t* r_host;
  cudaStream_t stream;
  bool mip;  // gsr_forward_mip: the 2D Mip filter of width kernel_size replaces the 0.3 dilation
  float kernel_size;
};
// what a backward takes besides the kernels' arguments (BwdArgs)
struct BwdHost {
  int64_t R;
  char *geom_buffer, *binning_buffer, *image_buffer;
  const float *dL_dpix, *dL_dpix_depth, *dL_dpix_median_depth, *dL_dpix_final_opacity, *background;
  // gsr_debug_projection_backward: the screen-space sums come from the caller instead of the compositing backward,
  // which is skipped along with its inputs
  const float* accum;
  int debug;
  cudaStream_t stream;
  bool mip;  // gsr_backward_mip: the backward of the Mip projection, which needs the input opacities
  float kernel_size;
  const float* opacities;
};

const char* forward_error(const FwdArgs& a) {
  if (a.P <= 0 || a.W <= 0 || a.H <= 0) return "gsr_forward: P, width and height must be positive";
  if (a.colors_precomp == nullptr && a.shs == nullptr && !a.fused) return "gsr_forward: need shs or colors_precomp";
  if (a.fused && (!a.f_dc || (a.M > 1 && !a.f_rest) || !a.scales || !a.rotations || a.M < 1)) return "gsr_forward_fused: need f_dc, f_rest, raw scales and rotations";
  if (a.cov3D_precomp == nullptr && (a.scales == nullptr || a.rotations == nullptr)) return "gsr_forward: need scales+rotations or cov3D_precomp";
  if (misaligned16(a.rotations)) return "gsr_forward: rotations must be 16-byte aligned";
  if (a.D < 0 || a.D > 3 || ((a.shs || a.fused) && (a.D + 1) * (a.D + 1) > a.M)) return "gsr_forward: sh degree / coefficient count mismatch";
  if (a.gx > 65535 || a.gy > 65535) return "gsr_forward: image too large";
  return nullptr;
}
const char* backward_error(const BwdArgs& a, const BwdHost& h) {
  if (!h.geom_buffer || (!h.accum && (!h.image_buffer || (!h.binning_buffer && h.R > 0)))) return "gsr_backward: missing state buffers";
  if (!h.background && !h.accum) return "gsr_backward: background must be a device pointer (backward.cu:586 reads it)";
  if (!a.cov3D_precomp && (!a.scales || !a.rotations))  // the backward recomputes cov3D from them
    return "gsr_backward: scales and rotations are required when cov3D_precomp is NULL";
  if (misaligned16(a.rotations) || misaligned16(a.dL_drot) || misaligned16(a.dL_dconic))
    return "gsr_backward: rotations, dL_drot and dL_dconic must be 16-byte aligned";
  return nullptr;
}

// sh_bulk / sh_rows of FwdArgs and BwdArgs.  `sh`: the SH pointers the projection kernel moves with TMA bulk copies,
// which need all of them 16-byte aligned -- f_dc / f_rest (and their gradients) as one block per CTA when fused, the
// [P,16,3] rows of shs (and dL_dsh) otherwise, and those only when all of them are given.
template <typename Args> void choose_sh_staging(Args& a, std::initializer_list<const float*> sh) {
  bool aligned = true, given = true;
  for (const float* p : sh) { aligned = aligned && !misaligned16(p); given = given && p; }
  a.sh_bulk = a.fused && a.M > 1 && aligned;
  a.sh_rows = !a.fused && a.M == 16 && given && aligned;
}

// first half of the forward: tile histogram reset, header (binning capacity `cap`), projection, tile scan
bool first_half(const FwdArgs& a, const FwdHost& h, GeomView g, ImageView im, unsigned long long cap) {
  const int T = a.gx * a.gy;
  if (!check(cudaMemsetAsync(im.tile_count, 0, sizeof(uint32_t) * T * SUBBINS, h.stream), "memset tile_count")) return false;
  launch_init_header(im.hdr, cap, h.stream);
  {
    Prof pf(kPreprocessFwd, h.stream);
    if (h.mip) launch_mip_preprocess_fwd(a, g, im, h.kernel_size, h.stream);
    else launch_preprocess_fwd(a, g, im, h.stream);
  }
  if (!stage_ok(h.debug, h.stream, "preprocess_fwd")) return false;
  { Prof pf(kTileScan, h.stream); launch_tile_scan(im, T, h.stream); }
  return stage_ok(h.debug, h.stream, "tile_scan");
}
// second half of the forward for a given binning capacity: scatter, per-tile sort, compositing
bool second_half(const FwdArgs& a, const FwdHost& h, GeomView g, ImageView im, long long cap) {
  char* bbuf = h.binning_alloc(h.binning_user, binning_bytes(cap));
  if (!bbuf) { set_last_error("gsr_forward: binning allocation failed"); return false; }
  BinView b = carve_binning(aligned_base(bbuf), cap);
  if (cap > 0) {
    { Prof pf(kScatter, h.stream); launch_scatter(a.P, a.gx, a.gx * a.gy, g, im, b, h.stream); }
    if (!stage_ok(h.debug, h.stream, "scatter")) return false;
    { Prof pf(kTileSort, h.stream); launch_tile_sort(a.gx * a.gy, g, im, b, h.stream); }
    if (!stage_ok(h.debug, h.stream, "tile_sort")) return false;
  }
  { Prof pf(kRenderFwd, h.stream); launch_render_fwd(a.W, a.H, a.gx, a.gy, im, b, g, fwd_tma_enabled(), h.out_color, h.out_depth, h.out_median_depth, h.out_opacity, h.stream); }
  return stage_ok(h.debug, h.stream, "render_fwd");
}

// Speculative exact mode (see above): the second half is already enqueued when the host blocks on the counts.
int64_t forward_speculative(const FwdArgs& a, const FwdHost& h, GeomView g, ImageView im, int dev, long long cap) {
  if (!first_half(a, h, g, im, (unsigned long long)cap)) return -1;
  long long* counts = t_spec.counts;
  if (!check(cudaMemcpyAsync(counts, &im.hdr->num_rendered, 16, cudaMemcpyDeviceToHost, h.stream), "read R")) return -1;
  if (!check(cudaEventRecord(t_spec.ev, h.stream), "read R (event)")) return -1;
  if (!second_half(a, h, g, im, cap)) return -1;
  if (!check(cudaEventSynchronize(t_spec.ev), "read R (sync)")) return -1;
  const long long binned = counts[0], ret = counts[1];
  if (h.r_host) *h.r_host = binned;
  hint_put(dev, a.P, a.W, a.H, binned);
  if (binned <= cap) {
    g_spec_hits.fetch_add(1, std::memory_order_relaxed);
    return ret;
  }
  // the guess was too small: redo the scan with the exact capacity, then the second half once more (stream order
  // keeps the abandoned launches, which only touched their own smaller buffer, ahead of the new ones)
  g_spec_redos.fetch_add(1, std::memory_order_relaxed);
  k_set_capacity<<<1, 1, 0, h.stream>>>(im.hdr, (unsigned long long)binned);
  { Prof pf(kTileScan, h.stream); launch_tile_scan(im, a.gx * a.gy, h.stream); }
  if (!stage_ok(h.debug, h.stream, "tile_scan (redo)")) return -1;
  return second_half(a, h, g, im, binned) ? ret : -1;
}

// Two counts: `binned` = tile instances that survive the exact tile culling (sizes the binning buffer) and the
// reference's num_rendered = sum of the rect areas (what the API returns in exact mode).
int64_t forward_impl(FwdArgs& a, const FwdHost& h) {
  a.gx = (a.W + TILE_X - 1) / TILE_X; a.gy = (a.H + TILE_Y - 1) / TILE_Y;
  if (const char* e = forward_error(a)) { set_last_error(e); return -1; }
  char* gbuf = h.geometry_alloc(h.geometry_user, geom_bytes(a.P));
  char* ibuf = h.image_alloc(h.image_user, image_bytes(a.W, a.H));
  if (!gbuf || !ibuf) return fail("gsr_forward", "scratch allocation failed");
  GeomView g = carve_geom(aligned_base(gbuf), a.P);
  ImageView im = carve_image(aligned_base(ibuf), a.W, a.H);
  a.focal_y = a.H / (2.0f * a.tan_fovy);  // rasterizer_impl.cu:225-226
  a.focal_x = a.W / (2.0f * a.tan_fovx);
  if (a.fused) choose_sh_staging(a, {a.f_dc, a.f_rest});
  else choose_sh_staging(a, {a.shs});
  if (h.r_capacity > 0) {  // pipelined mode: no host sync, the count arrives in *r_host
    if (!first_half(a, h, g, im, (unsigned long long)h.r_capacity)) return -1;
    if (h.r_host && !check(cudaMemcpyAsync(h.r_host, &im.hdr->num_rendered, 8, cudaMemcpyDeviceToHost, h.stream), "async R")) return -1;
    return second_half(a, h, g, im, h.r_capacity) ? h.r_capacity : -1;
  }
  // exact mode, from the second view of a shape on: speculate on the binning capacity
  int dev = 0;
  if (!h.debug && speculate_enabled() && cudaGetDevice(&dev) == cudaSuccess) {
    const long long hint = hint_get(dev, a.P, a.W, a.H);
    if (hint >= 0 && t_spec.ready(dev)) return forward_speculative(a, h, g, im, dev, spec_capacity(hint));
  }
  // exact mode: the one blocking read the reference also performs (rasterizer_impl.cu:284)
  if (!first_half(a, h, g, im, ~0ull)) return -1;
  long long counts[2] = {0, 0};  // {binned, rect-sum}: adjacent header fields
  if (!check(cudaMemcpyAsync(counts, &im.hdr->num_rendered, 16, cudaMemcpyDeviceToHost, h.stream), "read R")) return -1;
  if (!check(cudaStreamSynchronize(h.stream), "read R (sync)")) return -1;
  if (h.r_host) *h.r_host = counts[0];
  if (!h.debug && cudaGetDevice(&dev) == cudaSuccess) hint_put(dev, a.P, a.W, a.H, counts[0]);
  return second_half(a, h, g, im, counts[0]) ? counts[1] : -1;
}

int backward_impl(BwdArgs& a, const BwdHost& h) {
  if (a.P <= 0) return 0;
  if (const char* e = backward_error(a, h)) { set_last_error(e); return -1; }
  GeomView g = carve_geom(aligned_base(h.geom_buffer), a.P);
  if (a.radii == nullptr) a.radii = g.radii;  // rasterizer_impl.cu:381-384
  if (h.accum) {
    if (!check(cudaMemcpyAsync(g.grad, h.accum, sizeof(float) * GRAD_F * (size_t)a.P, cudaMemcpyDeviceToDevice, h.stream), "copy accum")) return -1;
  } else {
    if (!check(cudaMemsetAsync(g.grad, 0, sizeof(float) * GRAD_F * (size_t)a.P, h.stream), "memset grad")) return -1;
    if (h.R > 0) {
      const int gx = (a.W + TILE_X - 1) / TILE_X, gy = (a.H + TILE_Y - 1) / TILE_Y;
      ImageView im = carve_image(aligned_base(h.image_buffer), a.W, a.H);
      BinView b = carve_binning(aligned_base(h.binning_buffer), h.R);
      { Prof pf(kRenderBwd, h.stream); launch_render_bwd(a.W, a.H, gx, gy, h.background, im, b, g, h.dL_dpix, h.dL_dpix_depth,
                                                         h.dL_dpix_median_depth, h.dL_dpix_final_opacity, h.stream); }
      if (!stage_ok(h.debug, h.stream, "render_bwd")) return -1;
    }
  }
  a.focal_y = a.H / (2.0f * a.tan_fovy);
  a.focal_x = a.W / (2.0f * a.tan_fovx);
  if (a.fused) choose_sh_staging(a, {a.f_dc, a.f_rest, a.dL_df_dc, a.dL_df_rest});
  else choose_sh_staging(a, {a.shs, a.dL_dsh});
  {
    Prof pf(kPreprocessBwd, h.stream);
    if (h.mip) launch_mip_preprocess_bwd(a, g, h.opacities, h.kernel_size, h.stream);
    else launch_preprocess_bwd(a, g, h.stream);
  }
  return stage_ok(h.debug, h.stream, "preprocess_bwd") ? 0 : -1;
}
}  // namespace

int fail(const char* entry, const std::string& msg) {
  g_err = std::string(entry) + ": " + msg;
  return -1;
}
bool kernel_size_ok(float k) { return std::isfinite(k) && k >= 0.f; }

void launch_init_header(ImageHeader* hdr, unsigned long long cap, cudaStream_t st) {
  launch_high_priority(k_init_header, dim3(1), dim3(1), 0, st, hdr, cap);
}

}  // namespace gsr

using namespace gsr;

extern "C" {

int gsr_abi_version(void) { return GSR_ABI_VERSION; }
const char* gsr_last_error(void) { return g_err.c_str(); }
size_t gsr_geometry_bytes(int P) { return geom_bytes(P); }
size_t gsr_image_bytes(int width, int height) { return image_bytes(width, height); }
size_t gsr_binning_bytes(int64_t num_rendered) { return binning_bytes(num_rendered); }

int64_t gsr_forward(gsr_alloc_fn geometry_alloc, void* geometry_user, gsr_alloc_fn binning_alloc, void* binning_user,
                    gsr_alloc_fn image_alloc, void* image_user, int P, int D, int M, const float* background,
                    int width, int height, const float* means3D, const float* shs, const float* colors_precomp,
                    const float* opacities, const float* scales, float scale_modifier, const float* rotations,
                    const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
                    const float* cam_pos, float tan_fovx, float tan_fovy, int prefiltered, float* out_color,
                    float* out_depth, float* out_median_depth, float* out_opacity, int* radii, int debug,
                    int64_t r_capacity, int64_t* r_host, void* stream) {
  (void)background;  // the forward never reads it (no background blend, forward.cu:389-390; quirk 10)
  FwdArgs a{};
  a.P = P; a.D = D; a.M = M; a.W = width; a.H = height; a.prefiltered = prefiltered; a.radii_out = radii;
  a.means3D = means3D; a.shs = shs; a.colors_precomp = colors_precomp; a.opacities = opacities;
  a.scales = scales; a.rotations = rotations; a.cov3D_precomp = cov3D_precomp;
  a.view = viewmatrix; a.proj = projmatrix; a.campos = cam_pos;
  a.scale_modifier = scale_modifier; a.tan_fovx = tan_fovx; a.tan_fovy = tan_fovy;
  FwdHost h{};
  h.geometry_alloc = geometry_alloc; h.geometry_user = geometry_user; h.binning_alloc = binning_alloc;
  h.binning_user = binning_user; h.image_alloc = image_alloc; h.image_user = image_user;
  h.out_color = out_color; h.out_depth = out_depth; h.out_median_depth = out_median_depth; h.out_opacity = out_opacity;
  h.debug = debug; h.r_capacity = r_capacity; h.r_host = r_host; h.stream = (cudaStream_t)stream;
  return forward_impl(a, h);
}

int64_t gsr_forward_fused(gsr_alloc_fn geometry_alloc, void* geometry_user, gsr_alloc_fn binning_alloc,
                          void* binning_user, gsr_alloc_fn image_alloc, void* image_user, int P, int D, int M,
                          const float* background, int width, int height, const float* means3D, const float* f_dc,
                          const float* f_rest, const float* opacity_logits, const float* log_scales,
                          float scale_modifier, const float* raw_rotations, const float* viewmatrix,
                          const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy,
                          int prefiltered, float* out_color, float* out_depth, float* out_median_depth,
                          float* out_opacity, int* radii, int debug, int64_t r_capacity, int64_t* r_host, void* stream) {
  FwdArgs a{};
  a.P = P; a.D = D; a.M = M; a.W = width; a.H = height; a.prefiltered = prefiltered; a.radii_out = radii;
  a.fused = 1; a.means3D = means3D; a.f_dc = f_dc; a.f_rest = f_rest; a.opacities = opacity_logits;
  a.scales = log_scales; a.rotations = raw_rotations; a.view = viewmatrix; a.proj = projmatrix; a.campos = cam_pos;
  a.scale_modifier = scale_modifier; a.tan_fovx = tan_fovx; a.tan_fovy = tan_fovy;
  FwdHost h{};
  h.geometry_alloc = geometry_alloc; h.geometry_user = geometry_user; h.binning_alloc = binning_alloc;
  h.binning_user = binning_user; h.image_alloc = image_alloc; h.image_user = image_user;
  h.out_color = out_color; h.out_depth = out_depth; h.out_median_depth = out_median_depth; h.out_opacity = out_opacity;
  h.debug = debug; h.r_capacity = r_capacity; h.r_host = r_host; h.stream = (cudaStream_t)stream;
  return forward_impl(a, h);
}

int gsr_backward(int P, int D, int M, int64_t R, const float* background, int width, int height,
                 const float* means3D, const float* shs, const float* colors_precomp, const float* scales,
                 float scale_modifier, const float* rotations, const float* cov3D_precomp, const float* viewmatrix,
                 const float* projmatrix, const float* campos, float tan_fovx, float tan_fovy, const int* radii,
                 char* geom_buffer, char* binning_buffer, char* image_buffer, const float* dL_dpix,
                 const float* dL_dpix_depth, const float* dL_dpix_median_depth, const float* dL_dpix_final_opacity,
                 float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor, float* dL_ddepth,
                 float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot, int debug,
                 void* stream) {
  BwdArgs a{};
  a.P = P; a.D = D; a.M = M; a.W = width; a.H = height; a.radii = radii;
  a.means3D = means3D; a.shs = shs; a.colors_precomp = colors_precomp; a.scales = scales; a.rotations = rotations;
  a.cov3D_precomp = cov3D_precomp; a.view = viewmatrix; a.proj = projmatrix; a.campos = campos;
  a.scale_modifier = scale_modifier; a.tan_fovx = tan_fovx; a.tan_fovy = tan_fovy;
  a.dL_dmean2D = dL_dmean2D; a.dL_dconic = dL_dconic; a.dL_dopacity = dL_dopacity; a.dL_dcolor = dL_dcolor;
  a.dL_ddepth = dL_ddepth; a.dL_dmean3D = dL_dmean3D; a.dL_dcov3D = dL_dcov3D; a.dL_dsh = dL_dsh;
  a.dL_dscale = dL_dscale; a.dL_drot = dL_drot;
  BwdHost h{};
  h.R = R; h.geom_buffer = geom_buffer; h.binning_buffer = binning_buffer; h.image_buffer = image_buffer;
  h.dL_dpix = dL_dpix; h.dL_dpix_depth = dL_dpix_depth; h.dL_dpix_median_depth = dL_dpix_median_depth;
  h.dL_dpix_final_opacity = dL_dpix_final_opacity; h.background = background; h.debug = debug;
  h.stream = (cudaStream_t)stream;
  return backward_impl(a, h);
}

int64_t gsr_forward_mip(gsr_alloc_fn geometry_alloc, void* geometry_user, gsr_alloc_fn binning_alloc, void* binning_user,
                        gsr_alloc_fn image_alloc, void* image_user, int P, int D, int M, const float* background,
                        int width, int height, const float* means3D, const float* shs, const float* colors_precomp,
                        const float* opacities, const float* scales, float scale_modifier, const float* rotations,
                        const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
                        const float* cam_pos, float tan_fovx, float tan_fovy, int prefiltered, float* out_color,
                        float* out_depth, float* out_median_depth, float* out_opacity, int* radii, int debug,
                        int64_t r_capacity, int64_t* r_host, float kernel_size, void* stream) {
  if (!kernel_size_ok(kernel_size)) return fail("gsr_forward_mip", "kernel_size must be finite and >= 0");
  FwdArgs a{};
  a.P = P; a.D = D; a.M = M; a.W = width; a.H = height; a.prefiltered = prefiltered; a.radii_out = radii;
  a.means3D = means3D; a.shs = shs; a.colors_precomp = colors_precomp; a.opacities = opacities;
  a.scales = scales; a.rotations = rotations; a.cov3D_precomp = cov3D_precomp;
  a.view = viewmatrix; a.proj = projmatrix; a.campos = cam_pos;
  a.scale_modifier = scale_modifier; a.tan_fovx = tan_fovx; a.tan_fovy = tan_fovy;
  FwdHost h{};
  h.geometry_alloc = geometry_alloc; h.geometry_user = geometry_user; h.binning_alloc = binning_alloc;
  h.binning_user = binning_user; h.image_alloc = image_alloc; h.image_user = image_user;
  h.out_color = out_color; h.out_depth = out_depth; h.out_median_depth = out_median_depth; h.out_opacity = out_opacity;
  h.debug = debug; h.r_capacity = r_capacity; h.r_host = r_host; h.stream = (cudaStream_t)stream;
  h.mip = true; h.kernel_size = kernel_size;
  return forward_impl(a, h);
}

int gsr_backward_fused(int P, int D, int M, int64_t R, const float* background, int width, int height,
                       const float* means3D, const float* f_dc, const float* f_rest, const float* opacity_logits,
                       const float* log_scales, float scale_modifier, const float* raw_rotations,
                       const float* viewmatrix, const float* projmatrix, const float* campos, float tan_fovx,
                       float tan_fovy, const int* radii, char* geom_buffer, char* binning_buffer, char* image_buffer,
                       const float* dL_dpix, const float* dL_dpix_depth, const float* dL_dpix_median_depth,
                       const float* dL_dpix_final_opacity, float* dL_dmean2D, float* dL_dopacity_logit,
                       float* dL_dcolor, float* dL_dmean3D, float* dL_dcov3D, float* dL_df_dc, float* dL_df_rest,
                       float* dL_dlog_scale, float* dL_draw_rot, int debug, void* stream) {
  BwdArgs a{};
  a.P = P; a.D = D; a.M = M; a.W = width; a.H = height; a.radii = radii;
  a.fused = 1; a.means3D = means3D; a.f_dc = f_dc; a.f_rest = f_rest; a.opacities_raw = opacity_logits;
  a.scales = log_scales; a.rotations = raw_rotations; a.view = viewmatrix; a.proj = projmatrix; a.campos = campos;
  a.scale_modifier = scale_modifier; a.tan_fovx = tan_fovx; a.tan_fovy = tan_fovy;
  a.dL_dmean2D = dL_dmean2D; a.dL_dopacity = dL_dopacity_logit; a.dL_dcolor = dL_dcolor; a.dL_dmean3D = dL_dmean3D;
  a.dL_dcov3D = dL_dcov3D; a.dL_df_dc = dL_df_dc; a.dL_df_rest = dL_df_rest;
  a.dL_dscale = dL_dlog_scale; a.dL_drot = dL_draw_rot;
  BwdHost h{};
  h.R = R; h.geom_buffer = geom_buffer; h.binning_buffer = binning_buffer; h.image_buffer = image_buffer;
  h.dL_dpix = dL_dpix; h.dL_dpix_depth = dL_dpix_depth; h.dL_dpix_median_depth = dL_dpix_median_depth;
  h.dL_dpix_final_opacity = dL_dpix_final_opacity; h.background = background; h.debug = debug;
  h.stream = (cudaStream_t)stream;
  return backward_impl(a, h);
}

int gsr_backward_mip(int P, int D, int M, int64_t R, const float* background, int width, int height,
                     const float* means3D, const float* shs, const float* colors_precomp, const float* scales,
                     float scale_modifier, const float* rotations, const float* cov3D_precomp, const float* viewmatrix,
                     const float* projmatrix, const float* campos, float tan_fovx, float tan_fovy, const int* radii,
                     char* geom_buffer, char* binning_buffer, char* image_buffer, const float* dL_dpix,
                     const float* dL_dpix_depth, const float* dL_dpix_median_depth, const float* dL_dpix_final_opacity,
                     float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor, float* dL_ddepth,
                     float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot, int debug,
                     const float* opacities, float kernel_size, void* stream) {
  if (!kernel_size_ok(kernel_size)) return fail("gsr_backward_mip", "kernel_size must be finite and >= 0");
  if (P > 0 && !opacities) return fail("gsr_backward_mip", "opacities are required");
  BwdArgs a{};
  a.P = P; a.D = D; a.M = M; a.W = width; a.H = height; a.radii = radii;
  a.means3D = means3D; a.shs = shs; a.colors_precomp = colors_precomp; a.scales = scales; a.rotations = rotations;
  a.cov3D_precomp = cov3D_precomp; a.view = viewmatrix; a.proj = projmatrix; a.campos = campos;
  a.scale_modifier = scale_modifier; a.tan_fovx = tan_fovx; a.tan_fovy = tan_fovy;
  a.dL_dmean2D = dL_dmean2D; a.dL_dconic = dL_dconic; a.dL_dopacity = dL_dopacity; a.dL_dcolor = dL_dcolor;
  a.dL_ddepth = dL_ddepth; a.dL_dmean3D = dL_dmean3D; a.dL_dcov3D = dL_dcov3D; a.dL_dsh = dL_dsh;
  a.dL_dscale = dL_dscale; a.dL_drot = dL_drot;
  BwdHost h{};
  h.R = R; h.geom_buffer = geom_buffer; h.binning_buffer = binning_buffer; h.image_buffer = image_buffer;
  h.dL_dpix = dL_dpix; h.dL_dpix_depth = dL_dpix_depth; h.dL_dpix_median_depth = dL_dpix_median_depth;
  h.dL_dpix_final_opacity = dL_dpix_final_opacity; h.background = background; h.debug = debug;
  h.stream = (cudaStream_t)stream;
  h.mip = true; h.kernel_size = kernel_size; h.opacities = opacities;
  return backward_impl(a, h);
}

int gsr_depth2normal(const float* depth, int width, int height, float fx, float fy, float cx, float cy, float d_min,
                     float d_max, const float* rot, float* out, void* stream) {
  if (width <= 0 || height <= 0) return 0;
  if (!depth || !out) return fail("gsr_depth2normal", "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  {
    Prof pf(kDepth2Normal, st);
    // K^-1 entries computed on the host in float like torch.inverse of the float32 intrinsics
    launch_high_priority(k_depth2normal, dim3((width + 31) / 32, (height + 7) / 8), dim3(32, 8), 0, st, depth, width,
                         height, 1.0f / fx, 1.0f / fy, -cx / fx, -cy / fy, d_min, d_max, rot, out);
  }
  return launched("gsr_depth2normal");
}

int gsr_depth2point(const float* depth, int width, int height, float fx, float fy, float cx, float cy,
                    const float* cam_to_world, float* out, void* stream) {
  if (width <= 0 || height <= 0) return 0;
  if (!depth || !out) return fail("gsr_depth2point", "null pointer");
  k_depth2point<<<dim3((width + 31) / 32, (height + 7) / 8), dim3(32, 8), 0, (cudaStream_t)stream>>>(
      depth, width, height, 1.0f / fx, 1.0f / fy, -cx / fx, -cy / fy, cam_to_world, out);
  return launched("gsr_depth2point");
}

int gsr_debug_export(int P, int width, int height, int64_t R, const char* geom_buffer, const char* binning_buffer,
                     const char* image_buffer, uint32_t* point_list, uint32_t* ranges, uint32_t* n_contrib,
                     float* final_T, float* means2D, float* conic_opacity, float* depths, float* rgb, float* cov3D,
                     uint32_t* tiles_touched, unsigned char* clamped, void* stream) {
  if (!geom_buffer || !image_buffer || (R > 0 && !binning_buffer))
    return fail("gsr_debug_export", "missing state buffers");
  cudaStream_t st = (cudaStream_t)stream;
  GeomView g = carve_geom(aligned_base(const_cast<char*>(geom_buffer)), P);
  ImageView im = carve_image(aligned_base(const_cast<char*>(image_buffer)), width, height);
  BinView b = carve_binning(aligned_base(const_cast<char*>(binning_buffer)), R);
  if (P > 0) k_export_geom<<<blocks(P, 256), 256, 0, st>>>(P, g, means2D, conic_opacity, depths, rgb, cov3D, tiles_touched, clamped);
  if (R > 0 && point_list) k_export_list<<<blocks(R, 256), 256, 0, st>>>(R, im.hdr, b, point_list);
  const int N = width * height, T = ((width + TILE_X - 1) / TILE_X) * ((height + TILE_Y - 1) / TILE_Y);
  k_export_image<<<(max(N, T) + 255) / 256, 256, 0, st>>>(N, T, im, ranges, n_contrib, final_T);
  return launched("gsr_debug_export");
}

int gsr_debug_accumulator(int P, const char* geom_buffer, float* accum, void* stream) {
  if (!geom_buffer || !accum) return fail("gsr_debug_accumulator", "geom_buffer and accum are required");
  if (P <= 0) return 0;
  GeomView g = carve_geom(aligned_base(const_cast<char*>(geom_buffer)), P);
  return check(cudaMemcpyAsync(accum, g.grad, sizeof(float) * GRAD_F * (size_t)P, cudaMemcpyDeviceToDevice,
                               (cudaStream_t)stream), "gsr_debug_accumulator") ? 0 : -1;
}

int gsr_debug_projection_backward(int fused, int P, int D, int M, int width, int height, const float* means3D,
                                  const float* shs, const float* colors_precomp, const float* f_dc, const float* f_rest,
                                  const float* opacities, const float* scales, float scale_modifier,
                                  const float* rotations, const float* cov3D_precomp, const float* viewmatrix,
                                  const float* projmatrix, const float* campos, float tan_fovx, float tan_fovy,
                                  const int* radii, char* geom_buffer, const float* accum, float* dL_dmean2D,
                                  float* dL_dconic, float* dL_dopacity, float* dL_dcolor, float* dL_ddepth,
                                  float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh, float* dL_df_dc,
                                  float* dL_df_rest, float* dL_dscale, float* dL_drot, int debug, void* stream) {
  if (!accum) return fail("gsr_debug_projection_backward", "accum is required");
  BwdArgs a{};
  a.P = P; a.D = D; a.M = M; a.W = width; a.H = height; a.radii = radii;
  a.fused = fused != 0; a.means3D = means3D; a.scales = scales; a.rotations = rotations;
  a.view = viewmatrix; a.proj = projmatrix; a.campos = campos;
  a.scale_modifier = scale_modifier; a.tan_fovx = tan_fovx; a.tan_fovy = tan_fovy;
  a.dL_dmean2D = dL_dmean2D; a.dL_dconic = dL_dconic; a.dL_dopacity = dL_dopacity; a.dL_dcolor = dL_dcolor;
  a.dL_ddepth = dL_ddepth; a.dL_dmean3D = dL_dmean3D; a.dL_dcov3D = dL_dcov3D;
  a.dL_dscale = dL_dscale; a.dL_drot = dL_drot;
  if (fused) {  // the inputs and gradients only one variant has (gsr.h)
    a.f_dc = f_dc; a.f_rest = f_rest; a.opacities_raw = opacities; a.dL_df_dc = dL_df_dc; a.dL_df_rest = dL_df_rest;
  } else {
    a.shs = shs; a.colors_precomp = colors_precomp; a.cov3D_precomp = cov3D_precomp; a.dL_dsh = dL_dsh;
  }
  BwdHost h{};
  h.geom_buffer = geom_buffer; h.accum = accum; h.debug = debug; h.stream = (cudaStream_t)stream;
  return backward_impl(a, h);
}

int gsr_debug_projection_backward_mip(int P, int D, int M, int width, int height, const float* means3D,
                                      const float* shs, const float* colors_precomp, const float* opacities,
                                      const float* scales, float scale_modifier, const float* rotations,
                                      const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
                                      const float* campos, float tan_fovx, float tan_fovy, const int* radii,
                                      char* geom_buffer, const float* accum, float* dL_dmean2D, float* dL_dconic,
                                      float* dL_dopacity, float* dL_dcolor, float* dL_ddepth, float* dL_dmean3D,
                                      float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot,
                                      float kernel_size, int debug, void* stream) {
  const char* fn = "gsr_debug_projection_backward_mip";
  if (!accum) return fail(fn, "accum is required");
  if (!kernel_size_ok(kernel_size)) return fail(fn, "kernel_size must be finite and >= 0");
  if (P > 0 && !opacities) return fail(fn, "opacities are required");
  BwdArgs a{};
  a.P = P; a.D = D; a.M = M; a.W = width; a.H = height; a.radii = radii;
  a.means3D = means3D; a.shs = shs; a.colors_precomp = colors_precomp; a.scales = scales; a.rotations = rotations;
  a.cov3D_precomp = cov3D_precomp; a.view = viewmatrix; a.proj = projmatrix; a.campos = campos;
  a.scale_modifier = scale_modifier; a.tan_fovx = tan_fovx; a.tan_fovy = tan_fovy;
  a.dL_dmean2D = dL_dmean2D; a.dL_dconic = dL_dconic; a.dL_dopacity = dL_dopacity; a.dL_dcolor = dL_dcolor;
  a.dL_ddepth = dL_ddepth; a.dL_dmean3D = dL_dmean3D; a.dL_dcov3D = dL_dcov3D; a.dL_dsh = dL_dsh;
  a.dL_dscale = dL_dscale; a.dL_drot = dL_drot;
  BwdHost h{};
  h.geom_buffer = geom_buffer; h.accum = accum; h.debug = debug; h.stream = (cudaStream_t)stream;
  h.mip = true; h.kernel_size = kernel_size; h.opacities = opacities;
  return backward_impl(a, h);
}

int gsr_set_tile_order(int mode) { return set_tile_order(mode); }

int gsr_set_speculation(int on) { return g_speculate.exchange(on < 0 ? -1 : (on != 0)); }

int gsr_speculation_stats(int64_t* hits, int64_t* redos) {
  if (hits) *hits = g_spec_hits.load();
  if (redos) *redos = g_spec_redos.load();
  return 0;
}

int gsr_profile_enable(int on) {
  g_prof_on = on != 0;
  return 0;
}

int gsr_profile_read(float* ms, int* counts) {
  std::lock_guard<std::mutex> l(g_prof_mu);
  for (auto& r : g_prof) {
    float t = 0.f;
    if (cudaEventSynchronize(r.b) == cudaSuccess && cudaEventElapsedTime(&t, r.a, r.b) == cudaSuccess) {
      if (ms) ms[r.stage] += t;
      if (counts) counts[r.stage] += 1;
    }
    cudaEventDestroy(r.a);
    cudaEventDestroy(r.b);
  }
  g_prof.clear();
  return 0;
}

}  // extern "C"
