// VisualHull space carving (gaustudio/pipelines/initializers/mask.py:38-93): what the reference does with ~10 torch ops,
// a boolean gather and a nonzero host synchronisation per camera, then PyMCubes on the host.
//
//   k_hull_carve                 one thread per grid node: the node leaves at the first camera whose insideView test
//                                it fails (the reference's AND over every camera); camera records staged in shared
//                                memory in chunks, every mask read from one uint8 buffer at the camera's offset
//   k_mc_dense_count / _emit     marching cubes of the occupancy (gsr_mc.cuh), with the vertex of each crossing
//                                edge at `threshold` from its empty end and mapped to the world in double
//
// Grid node g = (i res + j) res + k is the reference's meshgrid point (lin[j], lin[i], lin[k]) - translate: i walks
// y, j walks x, k walks z, so the occupancy is the reference's `volume` array.  No atomics: the same inputs give the
// same bits.
#include "gsr_internal.cuh"
#include "../../include/gsr.h"
#include "gsr_mc.cuh"
#include <cmath>

namespace gsr {
namespace {

constexpr int CARVE_THREADS = 256;
constexpr int CAM_CHUNK = 128;  // camera records staged per round: 128 * (64 + 24) B = 11 KB

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

// ---- marching cubes of the occupancy (gsr_mc.cuh) ----
// Case bit k <=> corner k is empty, so the tables' triangles face the empty (carved) side in index space; the map to
// the world swaps the first two axes (the reference's axis swap), a reflection, so each triangle is written reversed.
struct Empty {
  const unsigned char* __restrict__ occ;
  __device__ bool operator()(long long g) const { return occ[g] == 0; }
};

// index coordinate q -> world: ((q / (res - 1)) (2 r) - r) - t, in double
__device__ __forceinline__ float to_world(double q, double den, double two_r, double r, double t) {
  return __double2float_rn(__dsub_rn(__dsub_rn(__dmul_rn(__ddiv_rn(q, den), two_r), r), t));
}
struct HullVertex {
  const unsigned char* __restrict__ occ;
  double threshold, radius, tx, ty, tz;
  __device__ void operator()(int res, long long g, const int c[3], const long long*, unsigned mask, float* v) const {
    // PyMCubes' interpolation (x2 - x1)(iso - f1)/(f2 - f1) + x1 with f in {0, 1}: iso from an empty start node,
    // 1 - iso from a filled one
    const double frac = occ[g] == 0 ? threshold : __dsub_rn(1.0, threshold);
    const double den = (double)(res - 1), two_r = __dmul_rn(2.0, radius);
    for (int a = 0; a < 3; a++) {
      if (!((mask >> a) & 1)) continue;
      double q[3] = {(double)c[0], (double)c[1], (double)c[2]};
      q[a] = __dadd_rn(q[a], frac);
      v[0] = to_world(q[1], den, two_r, radius, tx);  // world x walks the grid's second axis
      v[1] = to_world(q[0], den, two_r, radius, ty);
      v[2] = to_world(q[2], den, two_r, radius, tz);
      v += 3;
    }
  }
};

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
  return mc_dense<true>(fn, res, Empty{occ}, HullVertex{occ, threshold, radius, tx, ty, tz}, scratch_alloc,
                       scratch_user, vertex_alloc, vertex_user, face_alloc, face_user, n_faces, (cudaStream_t)stream);
}

}  // extern "C"
