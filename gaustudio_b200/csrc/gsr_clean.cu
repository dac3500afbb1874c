// Point-cloud cleaning on the device: what clean_point_cloud of gaustudio/scripts/extract_pcd.py:30-51 does with
// Open3D's PointCloud::RemoveStatisticalOutliers and a per-point Python loop over KDTreeFlann (remove_normal_outliers).
//
//   k_clean_box / k_clean_lattice      bounding box (min / max are order-free) -> a 2^21-per-axis integer lattice
//   k_clean_keys + radix sort          points sorted by the Morton code of their lattice cell: level l of the hierarchy
//   k_clean_gather                     (cells 2^l lattice units wide) is the key shifted right by 3l, one sort for all
//   k_clean_levels / k_clean_pick      the start level: the finest at which the median point's own cell holds
//                                      k/2 points (a density weighted by points: floaters alone in their cells do
//                                      not coarsen it)
//   k_clean_knn<MODE>                  one warp per query: exact k nearest (k <= 64), fused into its consumer
//   k_clean_partial / k_clean_stats    mean and Bessel std of the mean distances, in double, in a fixed order
//   k_clean_keep_stat / _keep_angle    the keep masks
//
// The neighbour search.  The best-k list is kept sorted by (squared distance, index) in two slots per lane (slot
// s = 32 e + lane).  The query scans Chebyshev shells r = 0, 1, ... of cells around its own cell at level l; after
// shell r every unscanned point lies more than r 2^l lattice units away on some axis, so the search stops once the
// k-th distance is below that.  A query whose shells 0..RMAX at level l do not settle it moves to level l + 2 (cells
// 4x wider) and keeps its list; points of cells it already scanned are skipped there, so an isolated point's search
// takes a few levels instead of a walk over empty cells.  Cells wholly beyond the current k-th distance are not read.
// Squared distances are formed in double from the float32 coordinates, (dx dx + dy dy) + dz dz without contraction:
// the selection is the float64 one, ties going to the lower index.
#include "gsr_internal.cuh"
#include "../../include/gsr.h"
#include <cub/cub.cuh>
#include <cmath>

namespace gsr {
namespace {

constexpr int KMAX = 64;
constexpr int BITS = 21;          // lattice cells per axis: 2^21; Morton keys of 63 bits
constexpr int TOP = BITS - 1;     // coarsest level: 2 cells per axis
constexpr int RMAX = 2;           // shells scanned at a level before moving up
constexpr int KNN_THREADS = 256;  // 8 queries per block
constexpr double MARGIN = 1e-9;   // lattice units: covers the rounding of (x - lo) * inv at |u| < 2^21
constexpr double SLACK = 1.0 + 1e-12;  // relative: covers the rounding of a box distance against a point's

struct Lattice {
  double lo[3];
  double inv;   // lattice cells per world unit
  int level;    // start level of the search
  int pad;
};

// ---- lattice ----
__global__ void __launch_bounds__(RED_THREADS) k_clean_box(int n, const float* __restrict__ xyz,
                                                          float* __restrict__ part) {
  __shared__ float red[2][3][RED_THREADS / 32];
  float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int i = blockIdx.x * RED_THREADS + threadIdx.x; i < n; i += RED_CTAS * RED_THREADS)
    for (int d = 0; d < 3; d++) {
      mn[d] = fminf(mn[d], xyz[3 * (size_t)i + d]);
      mx[d] = fmaxf(mx[d], xyz[3 * (size_t)i + d]);
    }
  for (int d = 0; d < 3; d++)
    for (int o = 16; o > 0; o >>= 1) {
      mn[d] = fminf(mn[d], __shfl_down_sync(0xffffffffu, mn[d], o));
      mx[d] = fmaxf(mx[d], __shfl_down_sync(0xffffffffu, mx[d], o));
    }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0)
    for (int d = 0; d < 3; d++) { red[0][d][warp] = mn[d]; red[1][d][warp] = mx[d]; }
  __syncthreads();
  if (threadIdx.x == 0)
    for (int d = 0; d < 3; d++) {
      float a = INFINITY, b = -INFINITY;
      for (int w = 0; w < RED_THREADS / 32; w++) { a = fminf(a, red[0][d][w]); b = fmaxf(b, red[1][d][w]); }
      part[6 * blockIdx.x + d] = a;
      part[6 * blockIdx.x + 3 + d] = b;
    }
}
__global__ void k_clean_lattice(const float* __restrict__ part, Lattice* __restrict__ lat) {
  float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int b = 0; b < RED_CTAS; b++)
    for (int d = 0; d < 3; d++) { mn[d] = fminf(mn[d], part[6 * b + d]); mx[d] = fmaxf(mx[d], part[6 * b + 3 + d]); }
  double ext = 0.0;
  for (int d = 0; d < 3; d++) {
    lat->lo[d] = mn[d];
    ext = fmax(ext, (double)mx[d] - (double)mn[d]);
  }
  lat->inv = ext > 0.0 ? (double)((1 << BITS) - 1) / ext : 1.0;
  lat->level = 0;
  lat->pad = 0;
}

// lattice coordinate of x on axis d (unrounded) and its cell; NaN / inf land in a valid cell
__device__ __forceinline__ double lat_u(const Lattice& L, int d, float x) {
  return __dmul_rn(__dsub_rn((double)x, L.lo[d]), L.inv);
}
__device__ __forceinline__ int lat_cell(double u) {
  return (int)fmin(fmax(floor(u), 0.0), (double)((1 << BITS) - 1));
}
__device__ __forceinline__ unsigned long long spread3(unsigned v) {
  unsigned long long x = v & 0x1fffffu;
  x = (x | x << 32) & 0x1f00000000ffffull;
  x = (x | x << 16) & 0x1f0000ff0000ffull;
  x = (x | x << 8) & 0x100f00f00f00f00full;
  x = (x | x << 4) & 0x10c30c30c30c30c3ull;
  x = (x | x << 2) & 0x1249249249249249ull;
  return x;
}
__device__ __forceinline__ unsigned long long morton(int x, int y, int z) {
  return spread3(x) << 2 | spread3(y) << 1 | spread3(z);
}

__global__ void k_clean_keys(int n, const float* __restrict__ xyz, const Lattice* __restrict__ lat,
                             unsigned long long* __restrict__ key, int* __restrict__ idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const Lattice L = *lat;
  int c[3];
  for (int d = 0; d < 3; d++) c[d] = lat_cell(lat_u(L, d, xyz[3 * (size_t)i + d]));
  key[i] = morton(c[0], c[1], c[2]);
  idx[i] = i;
}
// sorted points as (x, y, z, original index)
__global__ void k_clean_gather(int n, const int* __restrict__ order, const float* __restrict__ xyz,
                               float4* __restrict__ sp) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int i = order[j];
  sp[j] = make_float4(xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2], __int_as_float(i));
}
// The coarsest level is a single Chebyshev ring of 2 cells per axis; keys that differ above it share level TOP too.
__device__ __forceinline__ int shared_level(unsigned long long a, unsigned long long b) {
  const unsigned long long x = a ^ b;
  return x ? min((63 - __clzll(x)) / 3 + 1, TOP) : 0;
}
// hist[l]: points whose own cell first holds t or more points at level l.  In the sorted order, the cell of point i
// holds t points at level l iff some window of t consecutive keys around i shares a cell there, so that level is the
// least over the t windows holding i of the level at which the window's first and last keys agree.  Integer counts:
// the same on every run.
__global__ void k_clean_levels(int n, int t, const unsigned long long* __restrict__ key, int* __restrict__ hist) {
  __shared__ int h[BITS];
  if (threadIdx.x < BITS) h[threadIdx.x] = 0;
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    int level = TOP;
    for (int j = max(0, i - t + 1); j <= min(i, n - t); j++) level = min(level, shared_level(key[j], key[j + t - 1]));
    atomicAdd(&h[level], 1);
  }
  __syncthreads();
  if (threadIdx.x < BITS && h[threadIdx.x]) atomicAdd(hist + threadIdx.x, h[threadIdx.x]);
}
// The start level: the finest at which the median point's own cell holds t points.  A density weighted by points, so
// floaters, each alone in its cell, do not move it until they are half of the cloud.
__global__ void k_clean_pick(int n, const int* __restrict__ hist, Lattice* __restrict__ lat) {
  long long below = 0;
  int level = TOP;
  for (int l = 0; l <= TOP; l++) {
    below += hist[l];
    if (2 * below >= n) { level = l; break; }
  }
  lat->level = level;
}

// ---- the neighbour search ----
struct Best {
  double d[2];
  int i[2];
};
__device__ __forceinline__ bool key_less(double da, int ia, double db, int ib) {
  return da < db || (da == db && ia < ib);
}
// inserts (cd, ci), known to every lane, into the sorted list
__device__ __forceinline__ void insert(Best& b, double cd, int ci, int lane) {
  const unsigned lt0 = __ballot_sync(0xffffffffu, key_less(b.d[0], b.i[0], cd, ci));
  const unsigned lt1 = __ballot_sync(0xffffffffu, key_less(b.d[1], b.i[1], cd, ci));
  const int pos = __popc(lt0) + __popc(lt1);
  double pd0 = __shfl_up_sync(0xffffffffu, b.d[0], 1), pd1 = __shfl_up_sync(0xffffffffu, b.d[1], 1);
  int pi0 = __shfl_up_sync(0xffffffffu, b.i[0], 1), pi1 = __shfl_up_sync(0xffffffffu, b.i[1], 1);
  const double last_d = __shfl_sync(0xffffffffu, b.d[0], 31);
  const int last_i = __shfl_sync(0xffffffffu, b.i[0], 31);
  if (lane == 0) { pd1 = last_d; pi1 = last_i; }
  const int s0 = lane, s1 = 32 + lane;
  if (s0 > pos) { b.d[0] = pd0; b.i[0] = pi0; } else if (s0 == pos) { b.d[0] = cd; b.i[0] = ci; }
  if (s1 > pos) { b.d[1] = pd1; b.i[1] = pi1; } else if (s1 == pos) { b.d[1] = cd; b.i[1] = ci; }
}
__device__ __forceinline__ double sq_dist(float4 a, float4 b) {
  const double dx = __dsub_rn((double)a.x, (double)b.x), dy = __dsub_rn((double)a.y, (double)b.y),
               dz = __dsub_rn((double)a.z, (double)b.z);
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}
// first position in [0, n) whose key is >= v
__device__ __forceinline__ int lower_bound(const unsigned long long* __restrict__ key, int n, unsigned long long v) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(key + mid) < v) lo = mid + 1; else hi = mid;
  }
  return lo;
}

enum { MODE_KNN = 0, MODE_STAT = 1, MODE_ANGLE = 2, MODE_DIST2 = 3 };

// MODE_KNN:   out_idx[i*k + s] / out_d2[i*k + s], s < K = min(k, n): the K nearest of point i, itself included
// MODE_STAT:  out_val[i] = mean over those K of sqrt(d2)
// MODE_ANGLE: out_val[i] = mean over the K = min(k, n) - 1 nearest points other than i of acos(min(|n_i . n_j|, 1))
// MODE_DIST2: ((float*)out_val)[i] = float((d1 + d2 + d3) / 3) over the K = min(4, n) - 1 nearest points other than
//             i (k = 4), a missing neighbour counting as +inf: distCUDA2's contract.  (The float output shares
//             out_val so that the other modes keep their signature and code.)
template <int MODE>
__global__ void __launch_bounds__(KNN_THREADS, 3) k_clean_knn(int n, int k, const float4* __restrict__ sp,
                                                           const unsigned long long* __restrict__ key,
                                                           const Lattice* __restrict__ lat,
                                                           const float* __restrict__ normals, int* __restrict__ out_idx,
                                                           double* __restrict__ out_d2, double* __restrict__ out_val) {
  const int lane = threadIdx.x & 31;
  const int q = blockIdx.x * (KNN_THREADS / 32) + (threadIdx.x >> 5);
  if (q >= n) return;  // whole warps leave together
  const Lattice L = *lat;
  constexpr bool NOT_SELF = MODE == MODE_ANGLE || MODE == MODE_DIST2;
  const int K = NOT_SELF ? min(k, n) - 1 : min(k, n);
  const float4 Q = sp[q];
  const int self = __float_as_int(Q.w);
  const double uq[3] = {lat_u(L, 0, Q.x), lat_u(L, 1, Q.y), lat_u(L, 2, Q.z)};
  const int fq[3] = {lat_cell(uq[0]), lat_cell(uq[1]), lat_cell(uq[2])};
  const double h0 = 1.0 / L.inv;  // world units per lattice cell
  Best b;
  b.d[0] = b.d[1] = INFINITY;
  b.i[0] = b.i[1] = 0x7fffffff;
  int count = 0;
  double kd = INFINITY;  // the K-th squared distance, +inf until K points are held
  int ki = 0x7fffffff;
  int pl = -1, pr = 0, pc[3] = {0, 0, 0};  // the block of cells already scanned: level, radius, centre
  int l = L.level;
  bool done = K <= 0;
  while (!done) {
    const int ncell = 1 << (BITS - l);
    const int cq[3] = {fq[0] >> l, fq[1] >> l, fq[2] >> l};
    const double w = (double)(1 << l);  // cell width in lattice units
    for (int r = 0;; r++) {
      const int side = 2 * r + 1, total = side * side * side;
      for (int t0 = 0; t0 < total; t0 += 32) {
        const int t = t0 + lane;
        int a = 0, e = 0;
        double du2 = 0.0;
        if (t < total) {
          const int o[3] = {t / (side * side) - r, (t / side) % side - r, t % side - r};
          const bool shell = max(abs(o[0]), max(abs(o[1]), abs(o[2]))) == r;
          int c[3];
          bool in = shell;
          for (int d = 0; d < 3; d++) {
            c[d] = cq[d] + o[d];
            in = in && c[d] >= 0 && c[d] < ncell;
          }
          if (in) {
            // distance from the query to the cell's box in lattice units, less the rounding margin
            for (int d = 0; d < 3; d++) {
              const double lo = c[d] * w, hi = (c[d] + 1) * w;
              const double g = fmax(fmax(lo - uq[d], uq[d] - hi), 0.0);
              const double gm = fmax(g - MARGIN, 0.0) * h0;
              du2 += gm * gm;
            }
            if (!(count >= K && du2 > kd * SLACK)) {
              const unsigned long long base = morton(c[0], c[1], c[2]) << (3 * l);
              a = lower_bound(key, n, base);
              e = lower_bound(key, n, base + (1ull << (3 * l)));
            }
          }
        }
        unsigned todo = __ballot_sync(0xffffffffu, e > a);
        while (todo) {
          const int src = __ffs(todo) - 1;
          todo &= todo - 1;
          const int ca = __shfl_sync(0xffffffffu, a, src), ce = __shfl_sync(0xffffffffu, e, src);
          const double cdu2 = __shfl_sync(0xffffffffu, du2, src);
          if (count >= K && cdu2 > kd * SLACK) continue;  // the list has shrunk past this cell
          for (int j0 = ca; j0 < ce; j0 += 32) {
            const int j = j0 + lane;
            double cd = INFINITY;
            int ci = 0x7fffffff;
            bool ok = false;
            if (j < ce) {
              const float4 P = sp[j];
              ci = __float_as_int(P.w);
              ok = !(NOT_SELF && ci == self);
              if (ok && pl >= 0) {  // already scanned at level pl?
                bool inside = true;
                const float pp[3] = {P.x, P.y, P.z};
                for (int d = 0; d < 3; d++) inside = inside && abs((lat_cell(lat_u(L, d, pp[d])) >> pl) - pc[d]) <= pr;
                ok = !inside;
              }
              if (ok) cd = sq_dist(Q, P);
            }
            bool want = ok && (count < K || key_less(cd, ci, kd, ki));
            unsigned m = __ballot_sync(0xffffffffu, want);
            while (m) {
              const int s = __ffs(m) - 1;
              const double sd = __shfl_sync(0xffffffffu, cd, s);
              const int si = __shfl_sync(0xffffffffu, ci, s);
              insert(b, sd, si, lane);
              count++;
              if (count >= K) {
                const int ks = K - 1;
                kd = __shfl_sync(0xffffffffu, ks < 32 ? b.d[0] : b.d[1], ks & 31);
                ki = __shfl_sync(0xffffffffu, ks < 32 ? b.i[0] : b.i[1], ks & 31);
              }
              m &= ~(1u << s);
              want = want && (lane > s) && (count < K || key_less(cd, ci, kd, ki));
              m = __ballot_sync(0xffffffffu, want);
            }
          }
        }
      }
      // every unscanned point is more than r w lattice units away on some axis
      const double reach = fmax(r * w - MARGIN, 0.0) * h0;
      if (r >= ncell - 1 || (count >= K && kd * SLACK < reach * reach)) { done = true; break; }
      if (r >= RMAX && l + 2 <= TOP) {
        pl = l; pr = r;
        for (int d = 0; d < 3; d++) pc[d] = cq[d];
        l += 2;
        break;
      }
    }
  }
  const int orig = self;
  if (MODE == MODE_KNN) {
    for (int e = 0; e < 2; e++) {
      const int s = 32 * e + lane;
      if (s < K) {
        out_idx[(size_t)orig * k + s] = b.i[e];
        out_d2[(size_t)orig * k + s] = b.d[e];
      }
    }
    return;
  }
  if (MODE == MODE_DIST2) {
    double d[3];
    for (int s = 0; s < 3; s++) {
      const double ds = __shfl_sync(0xffffffffu, b.d[0], s);
      d[s] = s < K ? ds : INFINITY;  // slots >= K may hold entries shifted past the K-th
    }
    if (lane == 0) reinterpret_cast<float*>(out_val)[orig] = (float)(__dadd_rn(__dadd_rn(d[0], d[1]), d[2]) / 3.0);
    return;
  }
  double v = 0.0;
  for (int e = 0; e < 2; e++) {
    const int s = 32 * e + lane;
    if (s >= K) continue;
    if (MODE == MODE_STAT) {
      v += sqrt(b.d[e]);
    } else {
      const int j = b.i[e];
      // products of two float32 values are exact in double; |dot| is clamped to 1 (NaN stays NaN)
      const double dot = __dadd_rn(__dadd_rn(__dmul_rn((double)normals[3 * (size_t)orig], (double)normals[3 * (size_t)j]),
                                             __dmul_rn((double)normals[3 * (size_t)orig + 1],
                                                       (double)normals[3 * (size_t)j + 1])),
                                   __dmul_rn((double)normals[3 * (size_t)orig + 2], (double)normals[3 * (size_t)j + 2]));
      double x = fabs(dot);
      x = x > 1.0 ? 1.0 : x;
      v += acos(x);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (lane == 0) out_val[orig] = v / (double)K;  // K = 0: 0 / 0 = NaN, as np.mean([])
}

// ---- statistics of the mean distances ----
// which = 0: sum of avg (the reference sums avg > 0 only; avg >= 0, so the sums agree)
// which = 1: sum over avg > 0 of (avg - mean)^2
__global__ void __launch_bounds__(RED_THREADS) k_clean_partial(int n, const double* __restrict__ avg, int which,
                                                              const double* __restrict__ stats,
                                                              double* __restrict__ part) {
  __shared__ double red[RED_THREADS / 32];
  const double mean = which ? stats[0] : 0.0;
  double s = 0.0;
  for (int i = blockIdx.x * RED_THREADS + threadIdx.x; i < n; i += RED_CTAS * RED_THREADS) {
    const double a = avg[i];
    if (a > 0.0) s += which ? (a - mean) * (a - mean) : a;
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}
// which = 0: stats[0] = mean; which = 1: stats[1] = std (Bessel over n), stats[2] = mean + ratio std
__global__ void __launch_bounds__(RED_CTAS) k_clean_stats(int n, const double* __restrict__ part, int which,
                                                         double ratio, double* __restrict__ stats) {
  __shared__ double red[RED_CTAS / 32];
  const double v = block_sum(part[threadIdx.x], red);
  if (threadIdx.x != 0) return;
  if (which == 0) {
    stats[0] = v / (double)n;
  } else {
    const double sd = sqrt(v / (double)(n - 1));  // n = 1: 0 / 0 = NaN, and nothing is kept
    stats[1] = sd;
    stats[2] = stats[0] + ratio * sd;
  }
}
__global__ void k_clean_keep_stat(int n, const double* __restrict__ avg, const double* __restrict__ stats,
                                  unsigned char* __restrict__ keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double a = avg[i];
  keep[i] = a > 0.0 && a < stats[2];
}
__global__ void k_clean_keep_angle(int n, const double* __restrict__ mean_angle, double theta,
                                   unsigned char* __restrict__ keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  keep[i] = mean_angle[i] < theta;  // NaN: dropped
}

// The sorted grid of every query: scratch asked once.
struct Grid {
  float4* sp;
  unsigned long long* key;
  Lattice* lat;
  double* part;  // RED_CTAS partial sums
};
bool build_grid(const char* fn, int n, int k, const float* xyz, gsr_alloc_fn scratch_alloc, void* scratch_user,
                cudaStream_t st, Grid& g) {
  size_t sort_tmp = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                  (const int*)nullptr, (int*)nullptr, n, 0, 3 * BITS, st);
  unsigned long long *key, *key2;
  int *idx, *idx2, *hist;
  float* box;
  char* tmp;
  if (!carve_scratch(fn, scratch_alloc, scratch_user, [&](char*& p) {
        take(p, key, n);
        take(p, key2, n);
        take(p, idx, n);
        take(p, idx2, n);
        take(p, g.sp, n);
        take(p, box, RED_CTAS * 6);
        take(p, g.lat, 1);
        take(p, hist, BITS);
        take(p, g.part, RED_CTAS);
        take(p, tmp, sort_tmp);
      }))
    return false;
  g.key = key2;
  cudaMemsetAsync(hist, 0, BITS * sizeof(int), st);
  k_clean_box<<<RED_CTAS, RED_THREADS, 0, st>>>(n, xyz, box);
  k_clean_lattice<<<1, 1, 0, st>>>(box, g.lat);
  k_clean_keys<<<blocks(n, 256), 256, 0, st>>>(n, xyz, g.lat, key, idx);
  cub::DeviceRadixSort::SortPairs(tmp, sort_tmp, (const unsigned long long*)key, key2, (const int*)idx, idx2, n,
                                  0, 3 * BITS, st);
  k_clean_gather<<<blocks(n, 256), 256, 0, st>>>(n, idx2, xyz, g.sp);
  const int t = max(1, min((k + 1) / 2, n));  // the points a start cell should hold: half of the k sought
  k_clean_levels<<<blocks(n, 256), 256, 0, st>>>(n, t, key2, hist);
  k_clean_pick<<<1, 1, 0, st>>>(n, hist, g.lat);
  return true;
}
unsigned knn_blocks(int n) { return blocks(n, KNN_THREADS / 32); }

bool k_ok(const char* fn, int k) {
  if (k >= 1 && k <= KMAX) return true;
  fail(fn, "k must be in 1..64");
  return false;
}

}  // namespace
}  // namespace gsr

using namespace gsr;

extern "C" {

int gsr_clean_knn(int64_t n, const float* xyz, int k, gsr_alloc_fn scratch_alloc, void* scratch_user, int* index,
                  double* sq_dist, void* stream) {
  const char* fn = "gsr_clean_knn";
  if (!count_ok(fn, n, "n") || !k_ok(fn, k)) return -1;
  if (!xyz || !scratch_alloc || !index || !sq_dist) return fail(fn, "xyz, scratch_alloc, index and sq_dist are required");
  cudaStream_t st = (cudaStream_t)stream;
  Grid g;
  if (!build_grid(fn, (int)n, k, xyz, scratch_alloc, scratch_user, st, g)) return -1;
  k_clean_knn<MODE_KNN><<<knn_blocks((int)n), KNN_THREADS, 0, st>>>((int)n, k, g.sp, g.key, g.lat, nullptr, index,
                                                                     sq_dist, nullptr);
  return launched(fn);
}

int gsr_clean_statistical(int64_t n, const float* xyz, int k, double std_ratio, gsr_alloc_fn scratch_alloc,
                          void* scratch_user, double* avg_dist, double* stats, unsigned char* keep, void* stream) {
  const char* fn = "gsr_clean_statistical";
  if (!count_ok(fn, n, "n") || !k_ok(fn, k)) return -1;
  if (!(std_ratio > 0.0 && std_ratio < INFINITY)) return fail(fn, "std_ratio must be positive and finite");
  if (!xyz || !scratch_alloc || !avg_dist || !stats || !keep)
    return fail(fn, "xyz, scratch_alloc, avg_dist, stats and keep are required");
  cudaStream_t st = (cudaStream_t)stream;
  Grid g;
  if (!build_grid(fn, (int)n, k, xyz, scratch_alloc, scratch_user, st, g)) return -1;
  double* part = g.part;
  const int N = (int)n;
  k_clean_knn<MODE_STAT><<<knn_blocks(N), KNN_THREADS, 0, st>>>(N, k, g.sp, g.key, g.lat, nullptr, nullptr, nullptr,
                                                                avg_dist);
  k_clean_partial<<<RED_CTAS, RED_THREADS, 0, st>>>(N, avg_dist, 0, stats, part);
  k_clean_stats<<<1, RED_CTAS, 0, st>>>(N, part, 0, std_ratio, stats);
  k_clean_partial<<<RED_CTAS, RED_THREADS, 0, st>>>(N, avg_dist, 1, stats, part);
  k_clean_stats<<<1, RED_CTAS, 0, st>>>(N, part, 1, std_ratio, stats);
  k_clean_keep_stat<<<blocks(N, 256), 256, 0, st>>>(N, avg_dist, stats, keep);
  return launched(fn);
}

int gsr_clean_normal(int64_t n, const float* xyz, const float* normals, int k, double angle_threshold,
                     gsr_alloc_fn scratch_alloc, void* scratch_user, double* mean_angle, unsigned char* keep,
                     void* stream) {
  const char* fn = "gsr_clean_normal";
  if (!count_ok(fn, n, "n") || !k_ok(fn, k)) return -1;
  if (!(angle_threshold > -INFINITY && angle_threshold < INFINITY)) return fail(fn, "angle_threshold must be finite");
  if (!xyz || !normals || !scratch_alloc || !mean_angle || !keep)
    return fail(fn, "xyz, normals, scratch_alloc, mean_angle and keep are required");
  cudaStream_t st = (cudaStream_t)stream;
  Grid g;
  if (!build_grid(fn, (int)n, k, xyz, scratch_alloc, scratch_user, st, g)) return -1;
  k_clean_knn<MODE_ANGLE><<<knn_blocks((int)n), KNN_THREADS, 0, st>>>((int)n, k, g.sp, g.key, g.lat, normals, nullptr,
                                                                      nullptr, mean_angle);
  k_clean_keep_angle<<<blocks(n, 256), 256, 0, st>>>((int)n, mean_angle, angle_threshold, keep);
  return launched(fn);
}

int gsr_dist2(int64_t n, const float* xyz, gsr_alloc_fn scratch_alloc, void* scratch_user, float* dist2, void* stream) {
  const char* fn = "gsr_dist2";
  if (!count_ok(fn, n, "n")) return -1;
  if (!xyz || !scratch_alloc || !dist2) return fail(fn, "xyz, scratch_alloc and dist2 are required");
  cudaStream_t st = (cudaStream_t)stream;
  Grid g;
  if (!build_grid(fn, (int)n, 4, xyz, scratch_alloc, scratch_user, st, g)) return -1;
  k_clean_knn<MODE_DIST2><<<knn_blocks((int)n), KNN_THREADS, 0, st>>>((int)n, 4, g.sp, g.key, g.lat, nullptr, nullptr,
                                                                      nullptr, reinterpret_cast<double*>(dist2));
  return launched(fn);
}

}  // extern "C"
