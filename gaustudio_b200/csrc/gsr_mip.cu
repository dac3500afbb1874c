// Mip-Splatting's 3D smoothing filter (MipPointCloud.compute_3D_filter): one pass over all cameras instead of a torch
// loop of ~15 small kernels and two host-to-device copies per camera.
//   per camera c (records of gsr.h, gsr_mip_filter3d): p = x @ R + T, z' = max(p.z, 0.001),
//     u = p.x / z' fx + W/2, v = p.y / z' fy + H/2;  c sees x iff p.z > 0.2, -0.15 W <= u <= 1.15 W, -0.15 H <= v <= 1.15 H
//   d = min(100000, p.z over the cameras that see x); a Gaussian no camera sees gets the largest d of the seen ones
//   filter_3D = d / max_c fx * sqrt(0.2)
// The largest d and the largest fx are integer atomic maxima on float bits (both are positive), so the result does not
// depend on the order in which threads finish.
#include "../../include/gsr.h"
#include "gsr_internal.cuh"

namespace gsr {

namespace {

constexpr int F3_THREADS = 256;
constexpr int CAM_F = 16;       // floats per camera record: R (9, row-major), T (3), fx, fy, W, H
constexpr int CAM_CHUNK = 256;  // records staged in shared memory per round (16 KB)

// scratch[0]: bits of the largest d over the seen Gaussians, [1]: bits of the largest fx, [2]: seen Gaussians
__global__ void __launch_bounds__(F3_THREADS) k_mip_filter3d_min(int P, const float* __restrict__ xyz, int C,
                                                                 const float* __restrict__ cams, float* __restrict__ out,
                                                                 unsigned* __restrict__ scratch) {
  __shared__ float cs[CAM_CHUNK * CAM_F];
  const int i = blockIdx.x * F3_THREADS + threadIdx.x;
  // double: p.z can be much smaller than the terms it is summed from (a Gaussian close to a distant camera's image
  // plane), and float32 would then move d and the visibility decisions by more than a part in 1e6
  double x = 0.0, y = 0.0, z = 0.0;
  if (i < P) { x = xyz[3 * i]; y = xyz[3 * i + 1]; z = xyz[3 * i + 2]; }
  double d = 100000.0;
  bool seen = false;
  for (int c0 = 0; c0 < C; c0 += CAM_CHUNK) {
    const int n = min(CAM_CHUNK, C - c0);
    __syncthreads();  // the previous chunk has been read by every thread
    for (int k = threadIdx.x; k < n * CAM_F; k += F3_THREADS) {
      const float v = cams[(size_t)c0 * CAM_F + k];
      cs[k] = v;
      if (blockIdx.x == 0 && k % CAM_F == 12) atomicMax(&scratch[1], __float_as_uint(v));
    }
    __syncthreads();
    if (i < P) {
      for (int c = 0; c < n; c++) {
        const float* r = cs + c * CAM_F;  // every lane reads the same record: a broadcast
        const double px = x * r[0] + y * r[3] + z * r[6] + r[9];
        const double py = x * r[1] + y * r[4] + z * r[7] + r[10];
        const double pz = x * r[2] + y * r[5] + z * r[8] + r[11];
        const double iz = 1.0 / fmax(pz, 0.001), W = r[14], H = r[15];
        const double u = px * iz * r[12] + W * 0.5, v = py * iz * r[13] + H * 0.5;
        if (pz > 0.2 && u >= -0.15 * W && u <= 1.15 * W && v >= -0.15 * H && v <= 1.15 * H) {
          d = fmin(d, pz);
          seen = true;
        }
      }
    }
  }
  const float df = (float)d;
  if (i < P) out[i] = seen ? df : -1.f;  // -1: filled in by k_mip_filter3d_fill
  const unsigned dmax = __reduce_max_sync(0xffffffffu, seen ? __float_as_uint(df) : 0u);
  const unsigned cnt = __reduce_add_sync(0xffffffffu, seen ? 1u : 0u);
  if ((threadIdx.x & 31) == 0 && cnt) {
    atomicMax(&scratch[0], dmax);
    atomicAdd(&scratch[2], cnt);
  }
}

__global__ void k_mip_filter3d_fill(int P, float* __restrict__ out, const unsigned* __restrict__ scratch) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  float d = out[i];
  if (d < 0.f) d = __uint_as_float(scratch[0]);
  out[i] = d / __uint_as_float(scratch[1]) * 0.4472135955f;  // sqrt(0.2)
}

}  // namespace

}  // namespace gsr

using namespace gsr;

extern "C" int gsr_mip_filter3d(int P, const float* means3D, int n_cameras, const float* cameras, float* filter_3D,
                                unsigned int* scratch, void* stream) {
  const char* fn = "gsr_mip_filter3d";
  if (P < 0 || n_cameras < 0) return fail(fn, "P and n_cameras must be >= 0");
  if (P == 0) return 0;
  if (!means3D || !filter_3D || !scratch || (n_cameras > 0 && !cameras)) return fail(fn, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (cudaMemsetAsync(scratch, 0, 3 * sizeof(unsigned), st) != cudaSuccess) return fail(fn, "memset scratch failed");
  const unsigned nb = blocks(P, F3_THREADS);
  k_mip_filter3d_min<<<nb, F3_THREADS, 0, st>>>(P, means3D, n_cameras, cameras, filter_3D, scratch);
  k_mip_filter3d_fill<<<nb, F3_THREADS, 0, st>>>(P, filter_3D, scratch);
  return launched(fn);
}
