// Shape-as-Points meshing on the device: what gaustudio/models/sap.py (ShapeAsPoints.generate_mesh) and the DPSR of
// gaustudio/utils/graphics_utils.py do for the `--meshing sap` step of scripts/extract_pcd.py, there as ~40 torch ops,
// a scatter_add_ splat and skimage / cumcubes marching cubes on the host.
//
//   k_sap_sum / k_sap_center / k_sap_absmax / k_sap_scale / k_sap_points   c = mean, s = 1.2 max|x - c|, p in (0, 1)
//   k_sap_cells + radix sort + k_sap_gather     points bucketed by cell, stable in point index
//   k_sap_splat                                 per grid node: trilinear gather from its 8 neighbouring cells
//   k_sap_spectral                              one pass over the half spectrum: Phi = -i sum_d w_d G N_d / (-|w|^2 + 1e-6)
//   k_sap_interp / k_sap_offset / k_sap_psi     offset = mean of phi at the points; psi = tanh(-(phi - offset)/|fv0|/2)
//   k_mc_dense_count / _emit                    marching cubes of psi at 0 over the dense grid (gsr_mc.cuh)
//
// The forward and inverse FFTs between the splat and the spectral pass, and between the spectral pass and the shift,
// are cuFFT through torch.fft (gaustudio_b200/extract.py).  Every sum is formed in a fixed order (no float atomics),
// so the same inputs give the same bits.
#include "gsr_internal.cuh"
#include "../../include/gsr.h"
#include "gsr_mc.cuh"
#include <cmath>

namespace gsr {
namespace {

// ---- normalisation: transform = (c.x, c.y, c.z, s) as float32, the reference's float32 centre and scale ----
__global__ void __launch_bounds__(RED_THREADS) k_sap_sum(long long n, const float* __restrict__ xyz,
                                                        double* __restrict__ part) {
  __shared__ double red[RED_THREADS / 32];
  double s[3] = {0.0, 0.0, 0.0};
  for (long long i = (long long)blockIdx.x * RED_THREADS + threadIdx.x; i < n; i += (long long)RED_CTAS * RED_THREADS)
    for (int d = 0; d < 3; d++) s[d] += (double)xyz[3 * i + d];
  for (int d = 0; d < 3; d++) {
    const double v = block_sum(s[d], red);
    if (threadIdx.x == 0) part[3 * blockIdx.x + d] = v;
  }
}
__global__ void __launch_bounds__(RED_CTAS) k_sap_center(long long n, const double* __restrict__ part,
                                                        float* __restrict__ transform) {
  __shared__ double red[RED_CTAS / 32];
  for (int d = 0; d < 3; d++) {
    const double v = block_sum(part[3 * threadIdx.x + d], red);
    if (threadIdx.x == 0) transform[d] = (float)(v / (double)n);
  }
}
__global__ void __launch_bounds__(RED_THREADS) k_sap_absmax(long long n, const float* __restrict__ xyz,
                                                           const float* __restrict__ transform,
                                                           double* __restrict__ part) {
  __shared__ double red[RED_THREADS / 32];
  const double c[3] = {transform[0], transform[1], transform[2]};
  double m = 0.0;
  for (long long i = (long long)blockIdx.x * RED_THREADS + threadIdx.x; i < n; i += (long long)RED_CTAS * RED_THREADS)
    for (int d = 0; d < 3; d++) m = fmax(m, fabs((double)xyz[3 * i + d] - c[d]));
  m = block_max(m, red);
  if (threadIdx.x == 0) part[blockIdx.x] = m;
}
__global__ void __launch_bounds__(RED_CTAS) k_sap_scale(const double* __restrict__ part, float* __restrict__ transform) {
  __shared__ double red[RED_CTAS / 32];
  const double m = block_max(part[threadIdx.x], red);
  if (threadIdx.x == 0) transform[3] = (float)(1.2 * m);
}
// p = ((x - c) / s + 1) / 2 in float32, the reference's ShapeAsPoints.transform
__global__ void k_sap_points(long long n3, const float* __restrict__ xyz, const float* __restrict__ transform,
                             float* __restrict__ p) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n3) return;
  const float c = transform[i % 3], s = transform[3];
  p[i] = __fmul_rn(__fadd_rn(__fdiv_rn(__fsub_rn(xyz[i], c), s), 1.0f), 0.5f);
}

// ---- trilinear weights of point_rasterize / grid_interp, float32 operation by operation ----
// Along one axis a point in cell i0 = floor(p / cs) gives |p - (i0 + 1) cs| / cs to node i0 and |p - i0 cs| / cs to
// node i0 + 1 (mod res).  A coordinate on a node (p = i0 cs) gives all of it to i0.  i0 is clamped into the grid so
// that memory stays in bounds for any input; the Python layer refuses coordinates outside [0, 1).
struct AxisW {
  int i0;
  float w[2];
};
__device__ __forceinline__ AxisW axis_weights(float p, int res, float cs) {
  AxisW a;
  const int i = (int)floorf(__fdiv_rn(p, cs));
  a.i0 = min(max(i, 0), res - 1);
  const float x0 = __fmul_rn((float)i, cs), x1 = __fmul_rn(__fadd_rn((float)i, 1.0f), cs);
  a.w[0] = __fdiv_rn(fabsf(__fsub_rn(p, x1)), cs);
  a.w[1] = __fdiv_rn(fabsf(__fsub_rn(p, x0)), cs);
  return a;
}
__device__ __forceinline__ float cell_size(int res) { return __fdiv_rn(1.0f, (float)res); }

// ---- splat: points bucketed by cell (stable in point index), then one thread per node gathers ----
__global__ void k_sap_cells(long long n, const float* __restrict__ p, int res, unsigned* __restrict__ key,
                            int* __restrict__ idx, int* __restrict__ counts) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float cs = cell_size(res);
  const int x = axis_weights(p[3 * i], res, cs).i0, y = axis_weights(p[3 * i + 1], res, cs).i0,
            z = axis_weights(p[3 * i + 2], res, cs).i0;
  const unsigned k = ((unsigned)x * res + y) * res + z;
  key[i] = k;
  idx[i] = (int)i;
  atomicAdd(counts + k, 1);  // an integer count: the same on every run
}
__global__ void k_sap_gather(long long n, const int* __restrict__ order, const float* __restrict__ p,
                             const float* __restrict__ normals, float* __restrict__ sp, float* __restrict__ sn) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const long long i = order[j];
  for (int d = 0; d < 3; d++) {
    sp[3 * j + d] = p[3 * i + d];
    sn[3 * j + d] = normals[3 * i + d];
  }
}
// Node (x, y, z) takes, from the cell (x - ox, y - oy, z - oz) mod res for o = (ox, oy, oz) in x-major order and then
// from each point of that cell in point order, w_x[ox] * w_y[oy] * w_z[oz] * normal (the float32 product of the
// reference), summed in double.  A point on a node has weight 0 towards node i0 + 1 here, where the reference sends
// that 0 to i0 again: the sums are the same.
__global__ void __launch_bounds__(128) k_sap_splat(int res, const int* __restrict__ cell_start,
                                                   const float* __restrict__ sp, const float* __restrict__ sn,
                                                   float* __restrict__ grid) {
  const long long N = (long long)res * res * res;
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= N) return;
  const int x = (int)(g / ((long long)res * res)), y = (int)((g / res) % res), z = (int)(g % res);
  const float cs = cell_size(res);
  double ax_ = 0.0, ay_ = 0.0, az_ = 0.0;
  for (int o = 0; o < 8; o++) {
    const int ox = (o >> 2) & 1, oy = (o >> 1) & 1, oz = o & 1;
    const int cx = x - ox < 0 ? res - 1 : x - ox, cy = y - oy < 0 ? res - 1 : y - oy,
              cz = z - oz < 0 ? res - 1 : z - oz;
    const long long cell = ((long long)cx * res + cy) * res + cz;
    const int j1 = cell_start[cell + 1];
    for (int j = cell_start[cell]; j < j1; j++) {
      const AxisW ax = axis_weights(sp[3 * j], res, cs), ay = axis_weights(sp[3 * j + 1], res, cs),
                  az = axis_weights(sp[3 * j + 2], res, cs);
      const float w = __fmul_rn(__fmul_rn(ox ? ax.w[1] : ax.w[0], oy ? ay.w[1] : ay.w[0]), oz ? az.w[1] : az.w[0]);
      ax_ += (double)__fmul_rn(w, sn[3 * j]);
      ay_ += (double)__fmul_rn(w, sn[3 * j + 1]);
      az_ += (double)__fmul_rn(w, sn[3 * j + 2]);
    }
  }
  grid[g] = (float)ax_;
  grid[N + g] = (float)ay_;
  grid[2 * N + g] = (float)az_;
}

// ---- spectral solve on the half spectrum [res][res][res/2 + 1] ----
__device__ __forceinline__ int fftfreq(int i, int n) { return i < (n + 1) / 2 ? i : i - n; }

__global__ void __launch_bounds__(256) k_sap_spectral(int res, double sig, const float2* __restrict__ spec,
                                                      float2* __restrict__ phi_hat) {
  const int h = res / 2 + 1;
  const long long M = (long long)res * res * h;
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= M) return;
  const int i = (int)(q / ((long long)res * h)), j = (int)((q / h) % res), k = (int)(q % h);
  const int om[3] = {fftfreq(i, res), fftfreq(j, res), k};
  // spec_gaussian_filter: exp(-0.5 (sig 2 |w| / res)^2) in float64, rounded to float32
  const double dis = sqrt((double)om[0] * om[0] + (double)om[1] * om[1] + (double)om[2] * om[2]);
  const double a = sig * 2.0 * dis / (double)res;
  const float G = (float)exp(-0.5 * (a * a));
  float re = 0.0f, im = 0.0f, lap = 0.0f;
  for (int d = 0; d < 3; d++) {
    const float w = __fmul_rn(__fmul_rn((float)om[d], 2.0f), 3.14159265358979323846f);  // omega * 2 * pi in float32
    const float2 s = spec[d * M + q];
    // -i * (G N) * w = (Im(G N) w, -Re(G N) w)
    re = __fadd_rn(re, __fmul_rn(__fmul_rn(s.y, G), w));
    im = __fadd_rn(im, -__fmul_rn(__fmul_rn(s.x, G), w));
    lap = __fadd_rn(lap, __fmul_rn(w, w));
  }
  const float den = __fadd_rn(-lap, 1e-6f);
  phi_hat[q] = q == 0 ? make_float2(0.0f, 0.0f) : make_float2(__fdiv_rn(re, den), __fdiv_rn(im, den));
}

// ---- shift and scale ----
__global__ void __launch_bounds__(RED_THREADS) k_sap_interp(long long n, const float* __restrict__ p, int res,
                                                           const float* __restrict__ phi, double* __restrict__ part) {
  __shared__ double red[RED_THREADS / 32];
  const float cs = cell_size(res);
  double s = 0.0;
  for (long long i = (long long)blockIdx.x * RED_THREADS + threadIdx.x; i < n; i += (long long)RED_CTAS * RED_THREADS) {
    const AxisW ax = axis_weights(p[3 * i], res, cs), ay = axis_weights(p[3 * i + 1], res, cs),
                az = axis_weights(p[3 * i + 2], res, cs);
    double fv = 0.0;
    for (int o = 0; o < 8; o++) {
      const int ox = (o >> 2) & 1, oy = (o >> 1) & 1, oz = o & 1;
      const int x = ox ? (ax.i0 + 1 == res ? 0 : ax.i0 + 1) : ax.i0, y = oy ? (ay.i0 + 1 == res ? 0 : ay.i0 + 1) : ay.i0,
                z = oz ? (az.i0 + 1 == res ? 0 : az.i0 + 1) : az.i0;
      const float w = __fmul_rn(__fmul_rn(ax.w[ox], ay.w[oy]), az.w[oz]);
      fv += (double)__fmul_rn(phi[((long long)x * res + y) * res + z], w);
    }
    s += fv;
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}
__global__ void __launch_bounds__(RED_CTAS) k_sap_offset(long long n, const double* __restrict__ part,
                                                        double* __restrict__ offset) {
  __shared__ double red[RED_CTAS / 32];
  const double v = block_sum(part[threadIdx.x], red);
  if (threadIdx.x == 0) *offset = v / (double)n;
}
// psi = tanh(-(phi - offset) / |phi[0] - offset| * 0.5), the float32 steps of DPSR.forward and generate_mesh
__global__ void k_sap_psi(long long N, const float* __restrict__ phi, const double* __restrict__ offset,
                          float* __restrict__ psi) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= N) return;
  const float off = (float)*offset;
  const float fv0 = fabsf(__fsub_rn(phi[0], off));
  psi[g] = tanhf(__fmul_rn(__fdiv_rn(-__fsub_rn(phi[g], off), fv0), 0.5f));
}

// ---- marching cubes over the dense grid (gsr_mc.cuh): node g = (x res + y) res + z ----
// psi is positive outside the shape (on the side the input normals point; the grid corner has tanh(0.5)) and the
// tables' convention (case bit k <=> psi >= 0 at corner k, triangles facing psi > 0) gives outward faces.
struct Outside {
  const float* __restrict__ psi;
  __device__ bool operator()(long long g) const { return psi[g] >= 0.0f; }
};
struct SapVertex {
  const float* __restrict__ psi;
  const float* __restrict__ transform;
  __device__ void operator()(int res, long long g, const int c[3], const long long step[3], unsigned mask,
                             float* v) const {
    const float s = transform[3];
    const double f0 = psi[g];
    for (int a = 0; a < 3; a++) {
      if (!((mask >> a) & 1)) continue;
      const double f1 = psi[g + step[a]];
      const double t = __ddiv_rn(f0, __dsub_rn(f0, f1));
      for (int k = 0; k < 3; k++) {
        // index coordinate / res (mc_from_psr, real_scale=False), then ShapeAsPoints.transform(inverse=True)
        const float u = __double2float_rn(__ddiv_rn(k == a ? __dadd_rn((double)c[k], t) : (double)c[k], (double)res));
        v[k] = __fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(u, 2.0f), 1.0f), s), transform[k]);
      }
      v += 3;
    }
  }
};

int end_bit(long long cells) {
  int b = 1;
  while ((1LL << b) < cells) b++;
  return b;
}

}  // namespace
}  // namespace gsr

using namespace gsr;

extern "C" {

int gsr_sap_normalize(int64_t n, const float* xyz, gsr_alloc_fn scratch_alloc, void* scratch_user, float* points01,
                      float* transform, void* stream) {
  const char* fn = "gsr_sap_normalize";
  if (!count_ok(fn, n, "n")) return -1;
  if (!xyz || !points01 || !transform || !scratch_alloc)
    return fail(fn, "xyz, points01, transform and scratch_alloc are required");
  cudaStream_t st = (cudaStream_t)stream;
  double* part = reinterpret_cast<double*>(scratch_alloc(scratch_user, RED_CTAS * 3 * sizeof(double)));
  if (!part) return fail(fn, "scratch allocation failed");
  k_sap_sum<<<RED_CTAS, RED_THREADS, 0, st>>>(n, xyz, part);
  k_sap_center<<<1, RED_CTAS, 0, st>>>(n, part, transform);
  k_sap_absmax<<<RED_CTAS, RED_THREADS, 0, st>>>(n, xyz, transform, part);
  k_sap_scale<<<1, RED_CTAS, 0, st>>>(part, transform);
  k_sap_points<<<blocks(3 * n, 256), 256, 0, st>>>(3 * n, xyz, transform, points01);
  return launched(fn);
}

int gsr_sap_splat(int64_t n, const float* points01, const float* normals, int res, gsr_alloc_fn scratch_alloc,
                  void* scratch_user, float* grid, void* stream) {
  const char* fn = "gsr_sap_splat";
  if (!count_ok(fn, n, "n") || !res_ok(fn, res)) return -1;
  if (!points01 || !normals || !grid || !scratch_alloc)
    return fail(fn, "points01, normals, grid and scratch_alloc are required");
  cudaStream_t st = (cudaStream_t)stream;
  const long long cells = (long long)res * res * res;
  const int bits = end_bit(cells);
  size_t sort_tmp = 0, scan_tmp = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (const unsigned*)nullptr, (unsigned*)nullptr, (const int*)nullptr,
                                  (int*)nullptr, (int)n, 0, bits, st);
  cub::DeviceScan::ExclusiveSum(nullptr, scan_tmp, (int*)nullptr, (int)(cells + 1), st);
  int *start, *idx, *idx2;
  unsigned *key, *key2;
  float *sp, *sn;
  char* tmp;
  if (!carve_scratch(fn, scratch_alloc, scratch_user, [&](char*& p) {
        take(p, start, cells + 1);
        take(p, key, n);
        take(p, key2, n);
        take(p, idx, n);
        take(p, idx2, n);
        take(p, sp, 3 * n);
        take(p, sn, 3 * n);
        take(p, tmp, sort_tmp > scan_tmp ? sort_tmp : scan_tmp);
      }))
    return -1;
  cudaMemsetAsync(start, 0, (cells + 1) * 4, st);
  k_sap_cells<<<blocks(n, 256), 256, 0, st>>>(n, points01, res, key, idx, start);
  cub::DeviceScan::ExclusiveSum(tmp, scan_tmp, start, (int)(cells + 1), st);
  cub::DeviceRadixSort::SortPairs(tmp, sort_tmp, (const unsigned*)key, key2, (const int*)idx, idx2, (int)n, 0,
                                  bits, st);
  k_sap_gather<<<blocks(n, 256), 256, 0, st>>>(n, idx2, points01, normals, sp, sn);
  k_sap_splat<<<blocks(cells, 128), 128, 0, st>>>(res, start, sp, sn, grid);
  return launched(fn);
}

int gsr_sap_spectral(int res, double sig, const float* spectrum, float* phi_hat, void* stream) {
  const char* fn = "gsr_sap_spectral";
  if (!res_ok(fn, res)) return -1;
  if (!(sig > 0.0 && sig < 1e30)) return fail(fn, "sig must be positive and finite");
  if (!spectrum || !phi_hat) return fail(fn, "spectrum and phi_hat are required");
  const long long M = (long long)res * res * (res / 2 + 1);
  k_sap_spectral<<<blocks(M, 256), 256, 0, (cudaStream_t)stream>>>(res, sig, reinterpret_cast<const float2*>(spectrum),
                                                                   reinterpret_cast<float2*>(phi_hat));
  return launched(fn);
}

int gsr_sap_shift_scale(int64_t n, const float* points01, int res, const float* phi, gsr_alloc_fn scratch_alloc,
                        void* scratch_user, float* psi, void* stream) {
  const char* fn = "gsr_sap_shift_scale";
  if (!count_ok(fn, n, "n") || !res_ok(fn, res)) return -1;
  if (!points01 || !phi || !psi || !scratch_alloc) return fail(fn, "points01, phi, psi and scratch_alloc are required");
  cudaStream_t st = (cudaStream_t)stream;
  double* part = reinterpret_cast<double*>(scratch_alloc(scratch_user, (RED_CTAS + 1) * sizeof(double)));
  if (!part) return fail(fn, "scratch allocation failed");
  const long long N = (long long)res * res * res;
  k_sap_interp<<<RED_CTAS, RED_THREADS, 0, st>>>(n, points01, res, phi, part);
  k_sap_offset<<<1, RED_CTAS, 0, st>>>(n, part, part + RED_CTAS);
  k_sap_psi<<<blocks(N, 256), 256, 0, st>>>(N, phi, part + RED_CTAS, psi);
  return launched(fn);
}

int64_t gsr_sap_marching_cubes(int res, const float* psi, const float* transform, gsr_alloc_fn scratch_alloc,
                               void* scratch_user, gsr_alloc_fn vertex_alloc, void* vertex_user,
                               gsr_alloc_fn face_alloc, void* face_user, int64_t* n_faces, void* stream) {
  const char* fn = "gsr_sap_marching_cubes";
  if (!res_ok(fn, res)) return -1;
  if (!psi || !transform) return fail(fn, "psi and transform are required");
  if (!scratch_alloc || !vertex_alloc || !face_alloc || !n_faces)
    return fail(fn, "allocators and n_faces are required");
  return mc_dense<false>(fn, res, Outside{psi}, SapVertex{psi, transform}, scratch_alloc, scratch_user, vertex_alloc,
                        vertex_user, face_alloc, face_user, n_faces, (cudaStream_t)stream);
}

}  // extern "C"
