// C ABI of libgsr_b200 (include/gsr.h): buffer carving, stage orchestration, error reporting.
// Orchestration restates CudaRasterizer::Rasterizer::{forward,backward,markVisible}
// ($RAST/cuda_rasterizer/rasterizer_impl.cu:141-153, 198-343, 347-452) on top of the H100 kernels.
#include "../../include/gsr.h"
#include "gsr_internal.cuh"
#include <cmath>

#include <cstdio>
#include <cstdlib>
#include <atomic>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include <nvtx3/nvToolsExt.h>  // header-only NVTX v3: ranges cost nothing unless a profiler is attached

namespace gsr {

namespace {
thread_local std::string g_err;

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

template <typename T> inline void take(char*& p, T*& out, size_t count) {
  p = reinterpret_cast<char*>(align_up(reinterpret_cast<size_t>(p), 256));
  out = reinterpret_cast<T*>(p);
  p += count * sizeof(T);
}

bool check(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return true;
  g_err = std::string(what) + ": " + cudaGetErrorString(e);
  return false;
}
// CHECK_CUDA of the reference (auxiliary.h:166-173): with debug, synchronise and surface errors per stage
bool stage_ok(bool debug, cudaStream_t st, const char* what) {
  if (!check(cudaGetLastError(), what)) return false;
  if (debug && !check(cudaStreamSynchronize(st), what)) return false;
  return true;
}

// ---- optional per-stage timing (gsr_profile_*) ----
struct ProfRec { int stage; cudaEvent_t a, b; };
bool g_prof_on = false;
std::mutex g_prof_mu;
std::vector<ProfRec> g_prof;
const char* const kStageName[GSR_NUM_STAGES] = {"gsr:preprocess_fwd", "gsr:tile_scan", "gsr:scatter", "gsr:tile_sort",
                                                "gsr:render_fwd", "gsr:render_bwd", "gsr:preprocess_bwd",
                                                "gsr:depth2normal"};
// One per stage launch: an NVTX range (timeline tools) and, when gsr_profile_enable(1), a CUDA-event pair.
struct Prof {
  int stage; cudaStream_t st; cudaEvent_t a = nullptr, b = nullptr;
  Prof(int s, cudaStream_t t) : stage(s), st(t) {
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
inline char* aligned_base(char* p) { return reinterpret_cast<char*>(align_up(reinterpret_cast<size_t>(p), 256)); }

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

void launch_depth2normal(const float* depth, int W, int H, float fx, float fy, float cx, float cy, float dmin,
                         float dmax, const float* rot, float* out, cudaStream_t st) {
  dim3 blk(32, 8), grd((W + 31) / 32, (H + 7) / 8);
  // K^-1 entries computed on the host in float like torch.inverse of the float32 intrinsics
  launch_high_priority(k_depth2normal, grd, blk, 0, st, depth, W, H, 1.0f / fx, 1.0f / fy, -cx / fx, -cy / fy, dmin, dmax, rot, out);
}

void launch_depth2point(const float* depth, int W, int H, float fx, float fy, float cx, float cy, const float* c2w,
                        float* out, cudaStream_t st) {
  dim3 blk(32, 8), grd((W + 31) / 32, (H + 7) / 8);
  k_depth2point<<<grd, blk, 0, st>>>(depth, W, H, 1.0f / fx, 1.0f / fy, -cx / fx, -cy / fy, c2w, out);
}

void launch_debug_export(int P, int W, int H, long long R, GeomView g, BinView b, ImageView im,
                         uint32_t* point_list, uint32_t* ranges, uint32_t* n_contrib, float* final_T,
                         float* means2D, float* conic_opacity, float* depths, float* rgb, float* cov3D,
                         uint32_t* tiles_touched, unsigned char* clamped, cudaStream_t st) {
  if (P > 0) k_export_geom<<<(P + 255) / 256, 256, 0, st>>>(P, g, means2D, conic_opacity, depths, rgb, cov3D, tiles_touched, clamped);
  if (R > 0 && point_list) k_export_list<<<(unsigned)((R + 255) / 256), 256, 0, st>>>(R, im.hdr, b, point_list);
  const int N = W * H, T = ((W + TILE_X - 1) / TILE_X) * ((H + TILE_Y - 1) / TILE_Y);
  k_export_image<<<(max(N, T) + 255) / 256, 256, 0, st>>>(N, T, im, ranges, n_contrib, final_T);
}

}  // namespace gsr

using namespace gsr;

extern "C" {

int gsr_abi_version(void) { return GSR_ABI_VERSION; }
const char* gsr_last_error(void) { return g_err.c_str(); }
size_t gsr_geometry_bytes(int P) { return geom_bytes(P); }
size_t gsr_image_bytes(int width, int height) { return image_bytes(width, height); }
size_t gsr_binning_bytes(int64_t num_rendered) { return binning_bytes(num_rendered); }

static int64_t forward_impl(int fused, const float* f_dc, const float* f_rest, gsr_alloc_fn geometry_alloc, void* geometry_user, gsr_alloc_fn binning_alloc, void* binning_user,
                    gsr_alloc_fn image_alloc, void* image_user, int P, int D, int M, const float* background,
                    int width, int height, const float* means3D, const float* shs, const float* colors_precomp,
                    const float* opacities, const float* scales, float scale_modifier, const float* rotations,
                    const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
                    const float* cam_pos, float tan_fovx, float tan_fovy, int prefiltered, float* out_color,
                    float* out_depth, float* out_median_depth, float* out_opacity, int* radii, int debug,
                    int64_t r_capacity, int64_t* r_host, void* stream) {
  (void)background;  // the forward never reads it (no background blend, forward.cu:389-390; quirk 10)
  cudaStream_t st = (cudaStream_t)stream;
  const bool dbg = debug != 0;
  if (P <= 0 || width <= 0 || height <= 0) { g_err = "gsr_forward: P, width and height must be positive"; return -1; }
  if (colors_precomp == nullptr && shs == nullptr && !fused) { g_err = "gsr_forward: need shs or colors_precomp"; return -1; }
  if (fused && (!f_dc || (M > 1 && !f_rest) || !scales || !rotations || M < 1)) { g_err = "gsr_forward_fused: need f_dc, f_rest, raw scales and rotations"; return -1; }
  if (cov3D_precomp == nullptr && (scales == nullptr || rotations == nullptr)) { g_err = "gsr_forward: need scales+rotations or cov3D_precomp"; return -1; }
  if (D < 0 || D > 3 || ((shs || fused) && (D + 1) * (D + 1) > M)) { g_err = "gsr_forward: sh degree / coefficient count mismatch"; return -1; }
  const int gx = (width + TILE_X - 1) / TILE_X, gy = (height + TILE_Y - 1) / TILE_Y, T = gx * gy;
  if (gx > 65535 || gy > 65535) { g_err = "gsr_forward: image too large"; return -1; }

  char* gbuf = geometry_alloc(geometry_user, geom_bytes(P));
  char* ibuf = image_alloc(image_user, image_bytes(width, height));
  if (!gbuf || !ibuf) { g_err = "gsr_forward: scratch allocation failed"; return -1; }
  GeomView g = carve_geom(aligned_base(gbuf), P);
  ImageView im = carve_image(aligned_base(ibuf), width, height);

  FwdArgs a;
  a.P = P; a.D = D; a.M = M; a.W = width; a.H = height; a.gx = gx; a.gy = gy;
  a.means3D = means3D; a.shs = shs; a.colors_precomp = colors_precomp; a.opacities = opacities;
  a.scales = scales; a.rotations = rotations; a.cov3D_precomp = cov3D_precomp;
  a.view = viewmatrix; a.proj = projmatrix; a.campos = cam_pos;
  a.scale_modifier = scale_modifier; a.tan_fovx = tan_fovx; a.tan_fovy = tan_fovy;
  a.focal_y = height / (2.0f * tan_fovy);  // rasterizer_impl.cu:225-226
  a.focal_x = width / (2.0f * tan_fovx);
  a.prefiltered = prefiltered; a.radii_out = radii;
  a.fused = fused; a.f_dc = f_dc; a.f_rest = f_rest;
  a.sh_bulk = fused && M > 1 && ((reinterpret_cast<size_t>(f_dc) | reinterpret_cast<size_t>(f_rest)) & 15) == 0;
  a.sh_rows = !fused && shs && M == 16 && (reinterpret_cast<size_t>(shs) & 15) == 0;

  // exact mode, from the second view of a shape on: speculate on the binning capacity (see above)
  int dev = 0;
  long long spec_cap = 0;
  if (r_capacity <= 0 && !dbg && speculate_enabled() && cudaGetDevice(&dev) == cudaSuccess) {
    const long long h = hint_get(dev, P, width, height);
    if (h >= 0 && t_spec.ready(dev)) spec_cap = spec_capacity(h);
  }
  const unsigned long long cap0 = r_capacity > 0 ? (unsigned long long)r_capacity : (spec_cap > 0 ? (unsigned long long)spec_cap : ~0ull);
  if (!check(cudaMemsetAsync(im.tile_count, 0, sizeof(uint32_t) * T * SUBBINS, st), "memset tile_count")) return -1;
  launch_high_priority(k_init_header, dim3(1), dim3(1), 0, st, im.hdr, (unsigned long long)cap0);
  { Prof pf(0, st); launch_preprocess_fwd(a, g, im, st); }
  if (!stage_ok(dbg, st, "preprocess_fwd")) return -1;
  { Prof pf(1, st); launch_tile_scan(im, T, st); }
  if (!stage_ok(dbg, st, "tile_scan")) return -1;

  // second half of the forward for a given binning capacity: scatter, per-tile sort, compositing
  auto second_half = [&](long long cap) -> bool {
    char* bbuf = binning_alloc(binning_user, binning_bytes(cap));
    if (!bbuf) { g_err = "gsr_forward: binning allocation failed"; return false; }
    BinView b = carve_binning(aligned_base(bbuf), cap);
    if (cap > 0) {
      { Prof pf(2, st); launch_scatter(P, gx, T, g, im, b, st); }
      if (!stage_ok(dbg, st, "scatter")) return false;
      { Prof pf(3, st); launch_tile_sort(T, g, im, b, st); }
      if (!stage_ok(dbg, st, "tile_sort")) return false;
    }
    { Prof pf(4, st); launch_render_fwd(width, height, gx, gy, im, b, g, fwd_tma_enabled(), out_color, out_depth, out_median_depth, out_opacity, st); }
    return stage_ok(dbg, st, "render_fwd");
  };

  // Two counts: `binned` = tile instances that survive the exact tile culling (sizes the binning buffer) and the
  // reference's num_rendered = sum of the rect areas (what the API returns in exact mode).
  long long cap, ret;
  if (r_capacity > 0) {
    cap = ret = r_capacity;
    if (r_host && !check(cudaMemcpyAsync(r_host, &im.hdr->num_rendered, 8, cudaMemcpyDeviceToHost, st), "async R")) return -1;
  } else if (spec_cap > 0) {
    // speculative exact mode: the second half is already enqueued when the host blocks on the counts
    long long* counts = t_spec.counts;
    if (!check(cudaMemcpyAsync(counts, &im.hdr->num_rendered, 16, cudaMemcpyDeviceToHost, st), "read R")) return -1;
    if (!check(cudaEventRecord(t_spec.ev, st), "read R (event)")) return -1;
    if (!second_half(spec_cap)) return -1;
    if (!check(cudaEventSynchronize(t_spec.ev), "read R (sync)")) return -1;
    const long long binned = counts[0];
    ret = counts[1];
    if (r_host) *r_host = binned;
    hint_put(dev, P, width, height, binned);
    if (binned <= spec_cap) {
      g_spec_hits.fetch_add(1, std::memory_order_relaxed);
      return ret;
    }
    // the guess was too small: redo the scan with the exact capacity, then the second half once more (stream order
    // keeps the abandoned launches, which only touched their own smaller buffer, ahead of the new ones)
    g_spec_redos.fetch_add(1, std::memory_order_relaxed);
    k_set_capacity<<<1, 1, 0, st>>>(im.hdr, (unsigned long long)binned);
    { Prof pf(1, st); launch_tile_scan(im, T, st); }
    if (!stage_ok(dbg, st, "tile_scan (redo)")) return -1;
    cap = binned;
  } else {
    // exact mode: the one blocking read the reference also performs (rasterizer_impl.cu:284)
    long long counts[2] = {0, 0};  // {binned, rect-sum}: adjacent header fields
    if (!check(cudaMemcpyAsync(counts, &im.hdr->num_rendered, 16, cudaMemcpyDeviceToHost, st), "read R")) return -1;
    if (!check(cudaStreamSynchronize(st), "read R (sync)")) return -1;
    if (r_host) *r_host = counts[0];
    cap = counts[0];
    ret = counts[1];
    if (!dbg && cudaGetDevice(&dev) == cudaSuccess) hint_put(dev, P, width, height, cap);
  }
  if (!second_half(cap)) return -1;
  return ret;
}

static int backward_impl(int fused, const float* f_dc, const float* f_rest, const float* opacities_raw, float* dL_df_dc, float* dL_df_rest, int P, int D, int M, int64_t R, const float* background, int width, int height,
                 const float* means3D, const float* shs, const float* colors_precomp, const float* scales,
                 float scale_modifier, const float* rotations, const float* cov3D_precomp, const float* viewmatrix,
                 const float* projmatrix, const float* campos, float tan_fovx, float tan_fovy, const int* radii,
                 char* geom_buffer, char* binning_buffer, char* image_buffer, const float* dL_dpix,
                 const float* dL_dpix_depth, const float* dL_dpix_median_depth, const float* dL_dpix_final_opacity,
                 float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor, float* dL_ddepth,
                 float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot, int debug,
                 void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const bool dbg = debug != 0;
  if (P <= 0) return 0;
  if (!geom_buffer || !image_buffer || (!binning_buffer && R > 0)) { g_err = "gsr_backward: missing state buffers"; return -1; }
  if (!background) { g_err = "gsr_backward: background must be a device pointer (backward.cu:586 reads it)"; return -1; }
  if (!cov3D_precomp && (!scales || !rotations)) {  // the backward recomputes cov3D from them
    g_err = "gsr_backward: scales and rotations are required when cov3D_precomp is NULL";
    return -1;
  }
  const int gx = (width + TILE_X - 1) / TILE_X, gy = (height + TILE_Y - 1) / TILE_Y;
  GeomView g = carve_geom(aligned_base(geom_buffer), P);
  ImageView im = carve_image(aligned_base(image_buffer), width, height);
  BinView b = carve_binning(aligned_base(binning_buffer), R);
  if (radii == nullptr) radii = g.radii;  // rasterizer_impl.cu:381-384

  if (!check(cudaMemsetAsync(g.grad, 0, sizeof(float) * GRAD_F * (size_t)P, st), "memset grad")) return -1;
  if (R > 0) {
    { Prof pf(5, st); launch_render_bwd(width, height, gx, gy, background, im, b, g, dL_dpix, dL_dpix_depth, dL_dpix_median_depth,
                      dL_dpix_final_opacity, st); }
    if (!stage_ok(dbg, st, "render_bwd")) return -1;
  }
  BwdArgs a;
  a.P = P; a.D = D; a.M = M; a.W = width; a.H = height;
  a.means3D = means3D; a.shs = shs; a.colors_precomp = colors_precomp; a.scales = scales; a.rotations = rotations;
  a.cov3D_precomp = cov3D_precomp; a.view = viewmatrix; a.proj = projmatrix; a.campos = campos;
  a.scale_modifier = scale_modifier; a.tan_fovx = tan_fovx; a.tan_fovy = tan_fovy;
  a.focal_y = height / (2.0f * tan_fovy);
  a.focal_x = width / (2.0f * tan_fovx);
  a.radii = radii;
  a.dL_dmean2D = dL_dmean2D; a.dL_dconic = dL_dconic; a.dL_dopacity = dL_dopacity; a.dL_dcolor = dL_dcolor;
  a.dL_ddepth = dL_ddepth; a.dL_dmean3D = dL_dmean3D; a.dL_dcov3D = dL_dcov3D; a.dL_dsh = dL_dsh;
  a.dL_dscale = dL_dscale; a.dL_drot = dL_drot;
  a.fused = fused; a.f_dc = f_dc; a.f_rest = f_rest; a.opacities_raw = opacities_raw;
  a.dL_df_dc = dL_df_dc; a.dL_df_rest = dL_df_rest;
  a.sh_bulk = fused && M > 1 && ((reinterpret_cast<size_t>(f_dc) | reinterpret_cast<size_t>(f_rest) |
                                  reinterpret_cast<size_t>(dL_df_dc) | reinterpret_cast<size_t>(dL_df_rest)) & 15) == 0;
  a.sh_rows = !fused && shs && dL_dsh && M == 16 &&
              ((reinterpret_cast<size_t>(shs) | reinterpret_cast<size_t>(dL_dsh)) & 15) == 0;
  { Prof pf(6, st); launch_preprocess_bwd(a, g, st); }
  if (!stage_ok(dbg, st, "preprocess_bwd")) return -1;
  return 0;
}

int64_t gsr_forward(gsr_alloc_fn geometry_alloc, void* geometry_user, gsr_alloc_fn binning_alloc, void* binning_user,
                    gsr_alloc_fn image_alloc, void* image_user, int P, int D, int M, const float* background,
                    int width, int height, const float* means3D, const float* shs, const float* colors_precomp,
                    const float* opacities, const float* scales, float scale_modifier, const float* rotations,
                    const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
                    const float* cam_pos, float tan_fovx, float tan_fovy, int prefiltered, float* out_color,
                    float* out_depth, float* out_median_depth, float* out_opacity, int* radii, int debug,
                    int64_t r_capacity, int64_t* r_host, void* stream) {
  return forward_impl(0, nullptr, nullptr, geometry_alloc, geometry_user, binning_alloc, binning_user, image_alloc,
                      image_user, P, D, M, background, width, height, means3D, shs, colors_precomp, opacities, scales,
                      scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy,
                      prefiltered, out_color, out_depth, out_median_depth, out_opacity, radii, debug, r_capacity, r_host,
                      stream);
}

int64_t gsr_forward_fused(gsr_alloc_fn geometry_alloc, void* geometry_user, gsr_alloc_fn binning_alloc,
                          void* binning_user, gsr_alloc_fn image_alloc, void* image_user, int P, int D, int M,
                          const float* background, int width, int height, const float* means3D, const float* f_dc,
                          const float* f_rest, const float* opacity_logits, const float* log_scales,
                          float scale_modifier, const float* raw_rotations, const float* viewmatrix,
                          const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy,
                          int prefiltered, float* out_color, float* out_depth, float* out_median_depth,
                          float* out_opacity, int* radii, int debug, int64_t r_capacity, int64_t* r_host, void* stream) {
  return forward_impl(1, f_dc, f_rest, geometry_alloc, geometry_user, binning_alloc, binning_user, image_alloc,
                      image_user, P, D, M, background, width, height, means3D, nullptr, nullptr, opacity_logits,
                      log_scales, scale_modifier, raw_rotations, nullptr, viewmatrix, projmatrix, cam_pos, tan_fovx,
                      tan_fovy, prefiltered, out_color, out_depth, out_median_depth, out_opacity, radii, debug,
                      r_capacity, r_host, stream);
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
  return backward_impl(0, nullptr, nullptr, nullptr, nullptr, nullptr, P, D, M, R, background, width, height, means3D,
                       shs, colors_precomp, scales, scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix,
                       campos, tan_fovx, tan_fovy, radii, geom_buffer, binning_buffer, image_buffer, dL_dpix,
                       dL_dpix_depth, dL_dpix_median_depth, dL_dpix_final_opacity, dL_dmean2D, dL_dconic, dL_dopacity,
                       dL_dcolor, dL_ddepth, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, debug, stream);
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
  return backward_impl(1, f_dc, f_rest, opacity_logits, dL_df_dc, dL_df_rest, P, D, M, R, background, width, height,
                       means3D, nullptr, nullptr, log_scales, scale_modifier, raw_rotations, nullptr, viewmatrix,
                       projmatrix, campos, tan_fovx, tan_fovy, radii, geom_buffer, binning_buffer, image_buffer, dL_dpix,
                       dL_dpix_depth, dL_dpix_median_depth, dL_dpix_final_opacity, dL_dmean2D, nullptr, dL_dopacity_logit,
                       dL_dcolor, nullptr, dL_dmean3D, dL_dcov3D, nullptr, dL_dlog_scale, dL_draw_rot, debug, stream);
}

int gsr_mark_visible(int P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                     unsigned char* present, void* stream) {
  if (P <= 0) return 0;
  launch_mark_visible(P, means3D, viewmatrix, projmatrix, present, (cudaStream_t)stream);
  return check(cudaGetLastError(), "mark_visible") ? 0 : -1;
}

int gsr_depth2normal(const float* depth, int width, int height, float fx, float fy, float cx, float cy, float d_min,
                     float d_max, const float* rot, float* out, void* stream) {
  if (width <= 0 || height <= 0) return 0;
  { Prof pf(7, (cudaStream_t)stream); launch_depth2normal(depth, width, height, fx, fy, cx, cy, d_min, d_max, rot, out, (cudaStream_t)stream); }
  return check(cudaGetLastError(), "depth2normal") ? 0 : -1;
}

int gsr_depth2point(const float* depth, int width, int height, float fx, float fy, float cx, float cy,
                    const float* cam_to_world, float* out, void* stream) {
  if (width <= 0 || height <= 0) return 0;
  launch_depth2point(depth, width, height, fx, fy, cx, cy, cam_to_world, out, (cudaStream_t)stream);
  return check(cudaGetLastError(), "depth2point") ? 0 : -1;
}

int gsr_masked_bilateral(const float* depth, const unsigned char* mask, int width, int height, int d, float sigma_color,
                         float sigma_space, float* out_depth, unsigned char* out_mask, unsigned int* scratch,
                         void* stream) {
  if (width <= 0 || height <= 0) return 0;
  if (d < 1 || d > 15 || (d & 1) == 0) { g_err = "gsr_masked_bilateral: d must be odd, 1..15"; return -1; }
  if (!depth || !mask || !out_depth || !out_mask || !scratch) { g_err = "gsr_masked_bilateral: null pointer"; return -1; }
  // OpenCV: non-positive sigmas become 1; weights are evaluated in double and stored as float
  const double sc = sigma_color <= 0 ? 1.0 : (double)sigma_color, ss = sigma_space <= 0 ? 1.0 : (double)sigma_space;
  const double gauss_color = -0.5 / (sc * sc), gauss_space = -0.5 / (ss * ss);
  const int r = d / 2;
  SpaceKernel sk;
  for (int i = 0; i < 225; i++) sk.w[i] = 0.f;
  for (int dy = -r; dy <= r; dy++)
    for (int dx = -r; dx <= r; dx++) {
      const double rr = std::sqrt((double)dy * dy + (double)dx * dx);
      if (rr > r || (dy == 0 && dx == 0)) continue;
      sk.w[(dy + r) * (2 * r + 1) + dx + r] = (float)std::exp(rr * rr * gauss_space);
    }
  launch_masked_bilateral(depth, mask, width, height, r, (float)gauss_color, sk, out_depth, out_mask, scratch,
                          (cudaStream_t)stream);
  return check(cudaGetLastError(), "masked_bilateral") ? 0 : -1;
}

int gsr_extract_normals(const float* filtered_depth, const unsigned char* fg_mask, const float* opacity,
                        const float* median_depth, int width, int height, float fx, float fy, float cx, float cy,
                        const float* rot, float depth_limit, float opacity_min, float* cam_normals,
                        float* neg_world_normals, unsigned char* valid, void* stream) {
  if (width <= 0 || height <= 0) return 0;
  if (!filtered_depth || !fg_mask || !opacity || !median_depth || !rot || !neg_world_normals || !valid) {
    g_err = "gsr_extract_normals: null pointer"; return -1;
  }
  launch_extract_normals(filtered_depth, fg_mask, opacity, median_depth, width, height, fx, fy, cx, cy, rot, depth_limit,
                         opacity_min, cam_normals, neg_world_normals, valid, (cudaStream_t)stream);
  return check(cudaGetLastError(), "extract_normals") ? 0 : -1;
}

int gsr_normal_fusion_pass(int64_t n, const int64_t* ids, const float* normals, const float* confidences, int P,
                           const float* xyz, float cam_x, float cam_y, float cam_z, const float* mean_normals,
                           float threshold, float* sum_normals, float* sum_weights, unsigned char* touched,
                           void* stream) {
  if (n <= 0) return 0;
  if (!ids || !normals || !confidences || !xyz || !sum_normals || !sum_weights || P <= 0) {
    g_err = "gsr_normal_fusion_pass: null pointer"; return -1;
  }
  launch_fusion_pass((long long)n, reinterpret_cast<const long long*>(ids), normals, confidences, P, xyz, cam_x, cam_y,
                     cam_z, mean_normals, threshold, sum_normals, sum_weights, touched, (cudaStream_t)stream);
  return check(cudaGetLastError(), "normal_fusion_pass") ? 0 : -1;
}

int gsr_normal_fusion_mean(int P, const float* sum_normals, const float* sum_weights, float* mean_normals, void* stream) {
  if (P <= 0) return 0;
  launch_fusion_mean(P, sum_normals, sum_weights, mean_normals, (cudaStream_t)stream);
  return check(cudaGetLastError(), "normal_fusion_mean") ? 0 : -1;
}

int gsr_knn_grid(int n, int k, const float* points, const int* cell_start, const float* grid, int* out_index,
                 float* out_dist, void* stream) {
  if (n <= 0) return 0;
  if (!points || !cell_start || !grid || !out_index || !out_dist) { g_err = "gsr_knn_grid: null pointer"; return -1; }
  if (launch_knn_grid(n, k, points, cell_start, grid, out_index, out_dist, (cudaStream_t)stream) < 0) {
    g_err = "gsr_knn_grid: k must be 1, 4, 8, 10 or 16";
    return -1;
  }
  return check(cudaGetLastError(), "knn_grid") ? 0 : -1;
}

int gsr_adam_step(int n_groups, const gsr_adam_group* groups, double beta1, double beta2, double eps, int64_t step,
                  int decoupled, float grad_scale, int zero_grad, void* stream) {
  if (n_groups <= 0) return 0;
  if (!groups || n_groups > GSR_ADAM_MAX_GROUPS) { g_err = "gsr_adam_step: 1..16 groups"; return -1; }
  if (step < 1) { g_err = "gsr_adam_step: step counts from 1"; return -1; }
  for (int i = 0; i < n_groups; i++)
    if (groups[i].numel > 0 && (!groups[i].param || !groups[i].grad || !groups[i].exp_avg || !groups[i].exp_avg_sq)) {
      g_err = "gsr_adam_step: null tensor in a group"; return -1;
    }
  launch_adam(n_groups, groups, beta1, beta2, eps, (long long)step, decoupled, grad_scale, zero_grad, (cudaStream_t)stream);
  return check(cudaGetLastError(), "adam_step") ? 0 : -1;
}

int gsr_debug_export(int P, int width, int height, int64_t R, const char* geom_buffer, const char* binning_buffer,
                     const char* image_buffer, uint32_t* point_list, uint32_t* ranges, uint32_t* n_contrib,
                     float* final_T, float* means2D, float* conic_opacity, float* depths, float* rgb, float* cov3D,
                     uint32_t* tiles_touched, unsigned char* clamped, void* stream) {
  GeomView g = carve_geom(aligned_base(const_cast<char*>(geom_buffer)), P);
  ImageView im = carve_image(aligned_base(const_cast<char*>(image_buffer)), width, height);
  BinView b = carve_binning(aligned_base(const_cast<char*>(binning_buffer)), R);
  launch_debug_export(P, width, height, R, g, b, im, point_list, ranges, n_contrib, final_T, means2D, conic_opacity,
                      depths, rgb, cov3D, tiles_touched, clamped, (cudaStream_t)stream);
  return check(cudaGetLastError(), "debug_export") ? 0 : -1;
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
