// VisualHull space carving (gaustudio/pipelines/initializers/mask.py:38-93): what the reference does with ~10 torch ops,
// a boolean gather and a nonzero host synchronisation per camera, then PyMCubes on the host.
//
//   k_hull_carve                 one thread per grid node: the node leaves at the first camera whose insideView test
//                                it fails (the reference's AND over every camera); camera records staged in shared
//                                memory in chunks, every mask read from one uint8 buffer at the camera's offset
//   k_hull_count / k_hull_emit   marching cubes of the occupancy (gsr_mc_tables.cuh), with the vertex of each
//                                crossing edge at `threshold` from its empty end and mapped to the world in double
//
// Grid node g = (i res + j) res + k is the reference's meshgrid point (lin[j], lin[i], lin[k]) - translate: i walks
// y, j walks x, k walks z, so the occupancy is the reference's `volume` array.  No atomics: the same inputs give the
// same bits.
#include "gsr_internal.cuh"
#include "../../include/gsr.h"
#include "gsr_mc_tables.cuh"
#include <cub/cub.cuh>
#include <cmath>

namespace gsr {
namespace {

constexpr int CARVE_THREADS = 256;
constexpr int CAM_CHUNK = 128;  // camera records staged per round: 128 * (64 + 24) B = 11 KB
constexpr int MAX_RES = 512;

// np.linspace(start, stop, res)[i]: i * step + start (no contraction), the last node exactly stop
__device__ __forceinline__ double lin(int i, int res, double start, double step, double stop) {
  return i == res - 1 ? stop : __dadd_rn(__dmul_rn((double)i, step), start);
}

// the reference's Camera.insideView(x, mask) for one point, in double from float32 x and P (row-vector clip = [x 1] P)
__device__ __forceinline__ bool inside_view(const float x[3], const float* P, const long long* view,
                                            const unsigned char* __restrict__ masks) {
  double clip[4];
#pragma unroll
  for (int c = 0; c < 4; c++)
    clip[c] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn((double)x[0], (double)P[c]), __dmul_rn((double)x[1], (double)P[4 + c])),
                                  __dmul_rn((double)x[2], (double)P[8 + c])), (double)P[12 + c]);
  if (!(clip[2] > 0.0)) return false;
  const double nx = __ddiv_rn(clip[0], clip[3]), ny = __ddiv_rn(clip[1], clip[3]);
  if (!(nx >= -1.0 && nx <= 1.0 && ny >= -1.0 && ny <= 1.0)) return false;  // NaN and inf fail here
  const long long off = view[2];
  if (off < 0) return true;  // no mask: every pixel counts as inside
  const int W = (int)view[0], H = (int)view[1];
  const int px = min((int)__dmul_rn(__dmul_rn(__dadd_rn(nx, 1.0), 0.5), (double)W), W - 1);
  const int py = min((int)__dmul_rn(__dmul_rn(__dadd_rn(ny, 1.0), 0.5), (double)H), H - 1);
  return masks[off + (long long)py * W + px] != 0;
}

__global__ void __launch_bounds__(CARVE_THREADS) k_hull_carve(int res, double start, double step, double stop,
                                                              double tx, double ty, double tz, int C,
                                                              const float* __restrict__ proj,
                                                              const long long* __restrict__ views,
                                                              const unsigned char* __restrict__ masks,
                                                              unsigned char* __restrict__ occ) {
  __shared__ float sP[CAM_CHUNK * 16];
  __shared__ long long sV[CAM_CHUNK * 3];
  const long long N = (long long)res * res * res;
  const long long g = (long long)blockIdx.x * CARVE_THREADS + threadIdx.x;
  float x[3] = {0.f, 0.f, 0.f};
  bool filled = g < N;
  if (filled) {
    const int i = (int)(g / ((long long)res * res)), j = (int)((g / res) % res), k = (int)(g % res);
    x[0] = __double2float_rn(__dsub_rn(lin(j, res, start, step, stop), tx));
    x[1] = __double2float_rn(__dsub_rn(lin(i, res, start, step, stop), ty));
    x[2] = __double2float_rn(__dsub_rn(lin(k, res, start, step, stop), tz));
  }
  for (int c0 = 0; c0 < C; c0 += CAM_CHUNK) {
    // also the barrier after the previous chunk's reads; a block whose nodes are all carved stops here
    if (!__syncthreads_or(filled)) break;
    const int n = min(CAM_CHUNK, C - c0);
    for (int t = threadIdx.x; t < n * 16; t += CARVE_THREADS) sP[t] = proj[(size_t)c0 * 16 + t];
    for (int t = threadIdx.x; t < n * 3; t += CARVE_THREADS) sV[t] = views[(size_t)c0 * 3 + t];
    __syncthreads();
    for (int c = 0; c < n && filled; c++) filled = inside_view(x, sP + 16 * c, sV + 3 * c, masks);
  }
  if (g < N) occ[g] = filled ? 1 : 0;
}

// ---- marching cubes of the occupancy: node g is the base of cube g (all three indices < res - 1) ----
// Case bit k <=> corner k is empty, so the tables' triangles face the empty (carved) side in index space; the map to
// the world swaps the first two axes (the reference's axis swap), a reflection, so each triangle is written reversed.
__device__ __forceinline__ bool empty(unsigned char v) { return v == 0; }

__global__ void __launch_bounds__(128) k_hull_count(int res, const unsigned char* __restrict__ occ,
                                                    unsigned char* __restrict__ cube, unsigned char* __restrict__ edges,
                                                    int* __restrict__ fcount, int* __restrict__ vcount) {
  const long long N = (long long)res * res * res;
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g > N) return;
  if (g == N) { fcount[N] = 0; vcount[N] = 0; return; }
  const int c[3] = {(int)(g / ((long long)res * res)), (int)((g / res) % res), (int)(g % res)};
  const long long step[3] = {(long long)res * res, res, 1};
  const bool e0 = empty(occ[g]);
  unsigned mask = 0;
  for (int a = 0; a < 3; a++)
    if (c[a] + 1 < res && empty(occ[g + step[a]]) != e0) mask |= 1u << a;
  unsigned cs = 0;
  const bool full = c[0] + 1 < res && c[1] + 1 < res && c[2] + 1 < res;
  if (full)
    for (int k = 0; k < 8; k++)
      cs |= (unsigned)empty(occ[g + (k & 1) * step[0] + ((k >> 1) & 1) * step[1] + ((k >> 2) & 1) * step[2]]) << k;
  cube[g] = (unsigned char)cs;
  edges[g] = (unsigned char)mask;
  fcount[g] = full ? mc_ntri[cs] : 0;
  vcount[g] = __popc(mask);
}

// index coordinate q -> world: ((q / (res - 1)) (2 r) - r) - t, in double
__device__ __forceinline__ float to_world(double q, double den, double two_r, double r, double t) {
  return __double2float_rn(__dsub_rn(__dsub_rn(__dmul_rn(__ddiv_rn(q, den), two_r), r), t));
}

__global__ void __launch_bounds__(128) k_hull_emit(int res, const unsigned char* __restrict__ occ,
                                                   const unsigned char* __restrict__ cube,
                                                   const unsigned char* __restrict__ edges,
                                                   const int* __restrict__ vbase, const int* __restrict__ fbase,
                                                   double threshold, double radius, double tx, double ty, double tz,
                                                   float* __restrict__ verts, long long* __restrict__ faces) {
  const long long N = (long long)res * res * res;
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= N) return;
  const unsigned mask = edges[g], cs = cube[g];
  const int nt = mc_ntri[cs];
  if (!mask && !nt) return;
  const int c[3] = {(int)(g / ((long long)res * res)), (int)((g / res) % res), (int)(g % res)};
  const long long step[3] = {(long long)res * res, res, 1};
  if (mask) {
    // PyMCubes' interpolation (x2 - x1)(iso - f1)/(f2 - f1) + x1 with f in {0, 1}: iso from an empty start node,
    // 1 - iso from a filled one
    const double frac = empty(occ[g]) ? threshold : __dsub_rn(1.0, threshold);
    const double den = (double)(res - 1), two_r = __dmul_rn(2.0, radius);
    int vid = vbase[g];
    for (int a = 0; a < 3; a++) {
      if (!((mask >> a) & 1)) continue;
      double q[3] = {(double)c[0], (double)c[1], (double)c[2]};
      q[a] = __dadd_rn(q[a], frac);
      float* v = verts + 3 * (size_t)vid;
      v[0] = to_world(q[1], den, two_r, radius, tx);  // world x walks the grid's second axis
      v[1] = to_world(q[0], den, two_r, radius, ty);
      v[2] = to_world(q[2], den, two_r, radius, tz);
      vid++;
    }
  }
  long long fo = fbase[g];
  for (int t = 0; t < nt; t++, fo++)
    for (int j = 0; j < 3; j++) {
      const int e = mc_tri[cs][3 * t + j], c0 = mc_edge[e][0], a = mc_edge[e][2];
      const long long go = g + (c0 & 1) * step[0] + ((c0 >> 1) & 1) * step[1] + ((c0 >> 2) & 1) * step[2];
      faces[3 * fo + 2 - j] = vbase[go] + __popc(edges[go] & ((1u << a) - 1));
    }
}

__global__ void k_hull_counts(const int* __restrict__ vbase, const int* __restrict__ fbase, long long N,
                              long long* __restrict__ out) {
  out[0] = vbase[N];
  out[1] = fbase[N];
}

bool res_ok(const char* fn, int res) {
  if (res >= 2 && res <= MAX_RES) return true;
  fail(fn, "res must be in 2..512");
  return false;
}

}  // namespace
}  // namespace gsr

using namespace gsr;

extern "C" {

int gsr_hull_carve(int res, double radius, double tx, double ty, double tz, int n_cams, const float* proj,
                   const int64_t* views, const unsigned char* masks, unsigned char* occ, void* stream) {
  const char* fn = "gsr_hull_carve";
  if (!res_ok(fn, res)) return -1;
  if (!(radius > 0.0 && radius < 1e300)) return fail(fn, "radius must be positive and finite");
  if (!(std::isfinite(tx) && std::isfinite(ty) && std::isfinite(tz))) return fail(fn, "translate must be finite");
  if (n_cams < 0) return fail(fn, "n_cams must be >= 0");
  if (!occ || (n_cams > 0 && (!proj || !views))) return fail(fn, "occ, proj and views are required");
  const double start = -radius, stop = radius, step = (stop - start) / (double)(res - 1);
  const long long N = (long long)res * res * res;
  k_hull_carve<<<blocks(N, CARVE_THREADS), CARVE_THREADS, 0, (cudaStream_t)stream>>>(
      res, start, step, stop, tx, ty, tz, n_cams, proj, reinterpret_cast<const long long*>(views), masks, occ);
  return launched(fn);
}

int64_t gsr_hull_marching_cubes(int res, const unsigned char* occ, double threshold, double radius, double tx,
                                double ty, double tz, gsr_alloc_fn scratch_alloc, void* scratch_user,
                                gsr_alloc_fn vertex_alloc, void* vertex_user, gsr_alloc_fn face_alloc, void* face_user,
                                int64_t* n_faces, void* stream) {
  const char* fn = "gsr_hull_marching_cubes";
  if (!res_ok(fn, res)) return -1;
  if (!(threshold > 0.0 && threshold < 1.0)) return fail(fn, "threshold must be in (0, 1)");
  if (!(radius > 0.0 && radius < 1e300)) return fail(fn, "radius must be positive and finite");
  if (!(std::isfinite(tx) && std::isfinite(ty) && std::isfinite(tz))) return fail(fn, "translate must be finite");
  if (!occ) return fail(fn, "occ is required");
  if (!scratch_alloc || !vertex_alloc || !face_alloc || !n_faces)
    return fail(fn, "allocators and n_faces are required");
  cudaStream_t st = (cudaStream_t)stream;
  const long long N = (long long)res * res * res;
  size_t scan_tmp = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, scan_tmp, (int*)nullptr, (int)(N + 1), st);
  const size_t o_cube = 0, o_edges = align256(N), o_fb = o_edges + align256(N), o_vb = o_fb + align256((N + 1) * 4),
               o_rb = o_vb + align256((N + 1) * 4), o_tmp = o_rb + 256, total = o_tmp + align256(scan_tmp);
  char* s = scratch_alloc(scratch_user, total);
  if (!s) return fail(fn, "scratch allocation failed");
  unsigned char* cube = reinterpret_cast<unsigned char*>(s + o_cube);
  unsigned char* edges = reinterpret_cast<unsigned char*>(s + o_edges);
  int* fbase = reinterpret_cast<int*>(s + o_fb);
  int* vbase = reinterpret_cast<int*>(s + o_vb);
  long long* rb_dev = reinterpret_cast<long long*>(s + o_rb);
  k_hull_count<<<blocks(N + 1, 128), 128, 0, st>>>(res, occ, cube, edges, fbase, vbase);
  cub::DeviceScan::ExclusiveSum(s + o_tmp, scan_tmp, fbase, (int)(N + 1), st);
  cub::DeviceScan::ExclusiveSum(s + o_tmp, scan_tmp, vbase, (int)(N + 1), st);
  k_hull_counts<<<1, 1, 0, st>>>(vbase, fbase, N, rb_dev);
  long long rb[2];
  cudaMemcpyAsync(rb, rb_dev, sizeof(rb), cudaMemcpyDeviceToHost, st);
  if (launched(fn)) return -1;
  if (cudaStreamSynchronize(st) != cudaSuccess) { launched(fn); return -1; }
  const long long V = rb[0], F = rb[1];
  *n_faces = F;
  if (V == 0 && F == 0) return 0;
  char* verts = vertex_alloc(vertex_user, (size_t)V * 12);
  char* faces = face_alloc(face_user, (size_t)F * 24);
  if (!verts || !faces) return fail(fn, "output allocation failed");
  k_hull_emit<<<blocks(N, 128), 128, 0, st>>>(res, occ, cube, edges, vbase, fbase, threshold, radius, tx, ty, tz,
                                              reinterpret_cast<float*>(verts), reinterpret_cast<long long*>(faces));
  return launched(fn) ? -1 : V;
}

}  // extern "C"
