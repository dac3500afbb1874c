// Extraction post-pass on the device (SURVEY.md 8f row 2): what gaustudio/scripts/extract_pcd.py does to every
// rendered view right after the rasterizer -- and does on the CPU through OpenCV with a D2H/H2D round trip per view.
//
//   k_dilate_minmax    cv2.dilate of the invalid mask + nanmin/nanmax of the surviving depths  (extract_pcd.py:199-214)
//   k_bilateral        cv2.bilateralFilter on the normalised depth, de-normalise, restore     (extract_pcd.py:216-232)
//   k_extract_normals  depth2normal, -1 fill, normal2worldnormal, validity, negation          (extract_pcd.py:325-335)
//   k_fusion_pass      one weighted accumulation pass of normal_fusion                        (extract_pcd.py:117-136,143-165)
//   k_fusion_mean      mean = normalize(sum / weight)                                         (extract_pcd.py:139-140,167-168)
//
// All of it is streaming work: one thread per pixel (or per list entry), 4-13 bytes in, 1-28 bytes out, nothing
// that leaves HBM twice.  No host synchronisation anywhere (the depth range travels through two device words).
#include "gsr_internal.cuh"
#include "../../include/gsr.h"
#include <cmath>

namespace gsr {

// order-preserving float <-> uint map, so that atomicMin/atomicMax on the key order the floats
__device__ __forceinline__ unsigned f2key(float f) {
  const unsigned b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key2f(unsigned k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

__global__ void k_minmax_init(unsigned* scratch) { scratch[0] = 0xffffffffu; scratch[1] = 0u; }

// new_mask = every pixel of the (2r+1)^2 window that lies inside the image is valid (cv2.dilate of the invalid
// mask with its default border, which never contributes); min / max of depth over new_mask & !isnan.
__global__ void k_dilate_minmax(const float* __restrict__ depth, const unsigned char* __restrict__ mask, int W, int H,
                                int r, unsigned char* __restrict__ out_mask, unsigned* __restrict__ scratch) {
  const int u = blockIdx.x * blockDim.x + threadIdx.x, v = blockIdx.y * blockDim.y + threadIdx.y;
  unsigned kmin = 0xffffffffu, kmax = 0u;
  if (u < W && v < H) {
    bool ok = true;
    for (int dy = -r; dy <= r; dy++) {
      const int y = v + dy;
      if (y < 0 || y >= H) continue;
      for (int dx = -r; dx <= r; dx++) {
        const int x = u + dx;
        if (x < 0 || x >= W) continue;
        ok = ok && mask[(size_t)y * W + x] != 0;
      }
    }
    out_mask[(size_t)v * W + u] = ok;
    const float d = depth[(size_t)v * W + u];
    if (ok && d == d) kmin = kmax = f2key(d);
  }
  kmin = __reduce_min_sync(0xffffffffu, kmin);
  kmax = __reduce_max_sync(0xffffffffu, kmax);
  __shared__ unsigned smin[8], smax[8];
  const int warp = (threadIdx.y * blockDim.x + threadIdx.x) >> 5, lane = (threadIdx.y * blockDim.x + threadIdx.x) & 31;
  if (lane == 0) { smin[warp] = kmin; smax[warp] = kmax; }
  __syncthreads();
  if (warp == 0) {
    kmin = lane < 8 ? smin[lane] : 0xffffffffu;
    kmax = lane < 8 ? smax[lane] : 0u;
    kmin = __reduce_min_sync(0xffffffffu, kmin);
    kmax = __reduce_max_sync(0xffffffffu, kmax);
    if (lane == 0 && kmin != 0xffffffffu) { atomicMin(scratch, kmin); atomicMax(scratch + 1, kmax); }
  }
}

// OpenCV's borderInterpolate for BORDER_REFLECT_101: reflect again until the index is inside, 0 when n == 1.  One
// reflection is not enough once the radius reaches the image size (a 1-pixel-wide map, or d = 15 on a side under 8).
__device__ __forceinline__ int reflect101(int i, int n) {
  if (n == 1) return 0;
  while ((unsigned)i >= (unsigned)n) i = i < 0 ? -i : 2 * n - 2 - i;
  return i;
}

struct SpaceKernel { float w[225]; };  // (2r+1)^2 spatial weights of the bilateral filter, 0 outside the disc

// OpenCV's 32F bilateral filter on (depth - min) / (max - min) with invalid pixels at 0: disc support, centre weight
// 1, REFLECT_101 border; then filtered * (max - min) + min in separate roundings like the numpy expression.
__global__ void k_bilateral(const float* __restrict__ depth, const unsigned char* __restrict__ new_mask, int W, int H,
                            int r, float gauss_color, const __grid_constant__ SpaceKernel sk,
                            const unsigned* __restrict__ scratch, float* __restrict__ out) {
  const int u = blockIdx.x * blockDim.x + threadIdx.x, v = blockIdx.y * blockDim.y + threadIdx.y;
  if (u >= W || v >= H) return;
  const size_t pix = (size_t)v * W + u;
  const float d0 = depth[pix];
  const unsigned kmin = scratch[0];
  float res = d0;
  if (kmin != 0xffffffffu && new_mask[pix] && d0 == d0) {
    const float vmin = key2f(kmin), rng = __fsub_rn(key2f(scratch[1]), vmin);
    const float c = __fdiv_rn(__fsub_rn(d0, vmin), rng);
    float sum = c, wsum = 1.0f;
    const int dd = 2 * r + 1;
    for (int dy = -r; dy <= r; dy++) {
      const int y = reflect101(v + dy, H);
      for (int dx = -r; dx <= r; dx++) {
        const float ws = sk.w[(dy + r) * dd + dx + r];
        if (ws == 0.0f) continue;
        const int x = reflect101(u + dx, W);
        const size_t q = (size_t)y * W + x;
        const float dq = depth[q];
        const float nb = (new_mask[q] && dq == dq) ? __fdiv_rn(__fsub_rn(dq, vmin), rng) : 0.0f;
        const float diff = fabsf(nb - c);
        const float w = ws * expf(diff * diff * gauss_color);
        sum = fmaf(nb, w, sum);
        wsum += w;
      }
    }
    res = __fadd_rn(__fmul_rn(__fdiv_rn(sum, wsum), rng), vmin);
  }
  out[pix] = res;
}

__global__ void k_extract_normals(const float* __restrict__ depth, const unsigned char* __restrict__ fg,
                                  const float* __restrict__ opacity, const float* __restrict__ median_depth, int W,
                                  int H, float ifx, float ify, float ox, float oy, const float* __restrict__ rot,
                                  float depth_limit, float opacity_min, float* __restrict__ cam_normals,
                                  float* __restrict__ neg_world, unsigned char* __restrict__ valid) {
  const int u = blockIdx.x * blockDim.x + threadIdx.x, v = blockIdx.y * blockDim.y + threadIdx.y;
  if (u >= W || v >= H) return;
  const size_t pix = (size_t)v * W + u;
  float c0, c1, c2;
  if (!fg[pix] || !cross_normal(depth, u, v, W, H, ifx, ify, ox, oy, 1e-3f, 100000.0f, c0, c1, c2)) c0 = c1 = c2 = -1.f;
  // normal @ inverse(extrinsics[:3,:3]).t() -- applied to the -1 fill as well, as the reference does
  const float w0 = c0 * rot[0] + c1 * rot[3] + c2 * rot[6];
  const float w1 = c0 * rot[1] + c1 * rot[4] + c2 * rot[7];
  const float w2 = c0 * rot[2] + c1 * rot[5] + c2 * rot[8];
  const bool ok = (w0 + w1 + w2 > -3.0f) && median_depth[pix] < depth_limit && opacity[pix] > opacity_min;
  if (cam_normals) { cam_normals[3 * pix] = c0; cam_normals[3 * pix + 1] = c1; cam_normals[3 * pix + 2] = c2; }
  neg_world[3 * pix] = -w0; neg_world[3 * pix + 1] = -w1; neg_world[3 * pix + 2] = -w2;
  valid[pix] = ok;
}

__device__ __forceinline__ void red_add(float* p, float v) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}

__global__ void k_fusion_pass(long long n, const long long* __restrict__ ids, const float* __restrict__ normals,
                              const float* __restrict__ conf, int P, const float* __restrict__ xyz, float tx, float ty,
                              float tz, const float* __restrict__ mean, float thresh, float* __restrict__ sum_normals,
                              float* __restrict__ sum_weights, unsigned char* __restrict__ touched) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long id = ids[i];
  if (id < 0 || id >= P) return;
  const float nx = normals[3 * i], ny = normals[3 * i + 1], nz = normals[3 * i + 2];
  const float vx = tx - xyz[3 * id], vy = ty - xyz[3 * id + 1], vz = tz - xyz[3 * id + 2];
  const float dist = sqrtf(vx * vx + vy * vy + vz * vz);
  const float view_w = fabsf((vx / dist) * nx + (vy / dist) * ny + (vz / dist) * nz);
  const float w = conf[i] * view_w * (1.0f / (dist + 1e-6f));
  if (touched) touched[id] = 1;
  if (mean) {
    const float ex = nx - mean[3 * id], ey = ny - mean[3 * id + 1], ez = nz - mean[3 * id + 2];
    if (!(sqrtf(ex * ex + ey * ey + ez * ez) < thresh)) return;
  }
  red_add(sum_normals + 3 * id, nx * w);
  red_add(sum_normals + 3 * id + 1, ny * w);
  red_add(sum_normals + 3 * id + 2, nz * w);
  red_add(sum_weights + id, w);
}

__global__ void k_fusion_mean(int P, const float* __restrict__ sum_normals, const float* __restrict__ sum_weights,
                              float* __restrict__ mean) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  const float w = sum_weights[i];
  const float x = sum_normals[3 * i] / w, y = sum_normals[3 * i + 1] / w, z = sum_normals[3 * i + 2] / w;
  const float len = fmaxf(sqrtf(x * x + y * y + z * z), 1e-12f);  // F.normalize(p=2, eps=1e-12); NaN stays NaN
  mean[3 * i] = x / len; mean[3 * i + 1] = y / len; mean[3 * i + 2] = z / len;
}

}  // namespace gsr

// ---- k nearest neighbours on a uniform grid (neighbour search of extract_pcd.py:170-181, there scipy cKDTree on the host)
// One thread per query point (points are sorted by cell, so a warp's queries are neighbours in space and walk the same
// cells).  Rings of cells are scanned outwards; after the cube of radius r cells every point outside it is farther
// than r * cell_size, so the search stops once the k-th best distance is within that bound.
namespace gsr {
constexpr int KNN_MAX_K = 16;
template <int K>
__global__ void __launch_bounds__(128) k_knn_grid(int n, const float* __restrict__ pts, const int* __restrict__ cell_start,
                                                  const float* __restrict__ grid, int* __restrict__ out_index,
                                                  float* __restrict__ out_dist) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float ox = grid[0], oy = grid[1], oz = grid[2], inv_h = grid[3];
  const int dx = (int)grid[4], dy = (int)grid[5], dz = (int)grid[6];
  const float h = 1.0f / inv_h;
  const float qx = pts[3 * i], qy = pts[3 * i + 1], qz = pts[3 * i + 2];
  const int cx = min(dx - 1, max(0, (int)floorf((qx - ox) * inv_h)));
  const int cy = min(dy - 1, max(0, (int)floorf((qy - oy) * inv_h)));
  const int cz = min(dz - 1, max(0, (int)floorf((qz - oz) * inv_h)));
  float bd[K];
  int bi[K];
#pragma unroll
  for (int k = 0; k < K; k++) { bd[k] = 3.0e38f; bi[k] = -1; }
  const int rmax = max(dx, max(dy, dz));
  for (int r = 0; r <= rmax; r++) {
    // the shell of cells at Chebyshev distance exactly r from the query's cell
    auto scan = [&](int x, int y, int z) {
      const int c = (z * dy + y) * dx + x;
      for (int j = cell_start[c]; j < cell_start[c + 1]; j++) {
        const float ex = pts[3 * j] - qx, ey = pts[3 * j + 1] - qy, ez = pts[3 * j + 2] - qz;
        float d = ex * ex + ey * ey + ez * ez;
        if (d < bd[K - 1] || (d == bd[K - 1] && j < bi[K - 1])) {
          int id = j;
#pragma unroll
          for (int k = 0; k < K; k++) {  // insertion into the ascending list (ties: lower index first)
            const bool before = d < bd[k] || (d == bd[k] && id < bi[k]);
            const float td = before ? bd[k] : d;
            const int ti = before ? bi[k] : id;
            bd[k] = before ? d : bd[k];
            bi[k] = before ? id : bi[k];
            d = td; id = ti;
          }
        }
      }
    };
    for (int z = max(0, cz - r); z <= min(dz - 1, cz + r); z++)
      for (int y = max(0, cy - r); y <= min(dy - 1, cy + r); y++) {
        const bool face = (z == cz - r) || (z == cz + r) || (y == cy - r) || (y == cy + r);
        if (face || r == 0) {
          for (int x = max(0, cx - r); x <= min(dx - 1, cx + r); x++) scan(x, y, z);
        } else {  // interior row of the shell: only its two end cells
          if (cx - r >= 0) scan(cx - r, y, z);
          if (cx + r <= dx - 1) scan(cx + r, y, z);
        }
      }
    const float bound = (float)r * h;  // everything not scanned yet is farther than this
    if (bi[K - 1] >= 0 && bd[K - 1] <= bound * bound) break;
  }
#pragma unroll
  for (int k = 0; k < K; k++) {
    out_index[(size_t)i * K + k] = bi[k];
    out_dist[(size_t)i * K + k] = bi[k] >= 0 ? sqrtf(bd[k]) : __int_as_float(0x7f800000);
  }
}

}  // namespace gsr

using namespace gsr;

extern "C" {

int gsr_masked_bilateral(const float* depth, const unsigned char* mask, int width, int height, int d, float sigma_color,
                         float sigma_space, float* out_depth, unsigned char* out_mask, unsigned int* scratch,
                         void* stream) {
  if (width <= 0 || height <= 0) return 0;
  if (d < 1 || d > 15 || (d & 1) == 0) return fail("gsr_masked_bilateral", "d must be odd, 1..15");
  if (!depth || !mask || !out_depth || !out_mask || !scratch) return fail("gsr_masked_bilateral", "null pointer");
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
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 blk(32, 8), grd((width + 31) / 32, (height + 7) / 8);
  k_minmax_init<<<1, 1, 0, st>>>(scratch);
  k_dilate_minmax<<<grd, blk, 0, st>>>(depth, mask, width, height, r, out_mask, scratch);
  k_bilateral<<<grd, blk, 0, st>>>(depth, out_mask, width, height, r, (float)gauss_color, sk, scratch, out_depth);
  return launched("gsr_masked_bilateral");
}

int gsr_extract_normals(const float* filtered_depth, const unsigned char* fg_mask, const float* opacity,
                        const float* median_depth, int width, int height, float fx, float fy, float cx, float cy,
                        const float* rot, float depth_limit, float opacity_min, float* cam_normals,
                        float* neg_world_normals, unsigned char* valid, void* stream) {
  if (width <= 0 || height <= 0) return 0;
  if (!filtered_depth || !fg_mask || !opacity || !median_depth || !rot || !neg_world_normals || !valid)
    return fail("gsr_extract_normals", "null pointer");
  const dim3 blk(32, 8), grd((width + 31) / 32, (height + 7) / 8);
  k_extract_normals<<<grd, blk, 0, (cudaStream_t)stream>>>(filtered_depth, fg_mask, opacity, median_depth, width, height,
                                                            1.0f / fx, 1.0f / fy, -cx / fx, -cy / fy, rot, depth_limit,
                                                            opacity_min, cam_normals, neg_world_normals, valid);
  return launched("gsr_extract_normals");
}

int gsr_normal_fusion_pass(int64_t n, const int64_t* ids, const float* normals, const float* confidences, int P,
                           const float* xyz, float cam_x, float cam_y, float cam_z, const float* mean_normals,
                           float threshold, float* sum_normals, float* sum_weights, unsigned char* touched,
                           void* stream) {
  if (n <= 0) return 0;
  if (!ids || !normals || !confidences || !xyz || !sum_normals || !sum_weights || P <= 0)
    return fail("gsr_normal_fusion_pass", "null pointer");
  k_fusion_pass<<<blocks(n, 256), 256, 0, (cudaStream_t)stream>>>(
      (long long)n, reinterpret_cast<const long long*>(ids), normals, confidences, P, xyz, cam_x, cam_y, cam_z,
      mean_normals, threshold, sum_normals, sum_weights, touched);
  return launched("gsr_normal_fusion_pass");
}

int gsr_normal_fusion_mean(int P, const float* sum_normals, const float* sum_weights, float* mean_normals, void* stream) {
  if (P <= 0) return 0;
  k_fusion_mean<<<blocks(P, 256), 256, 0, (cudaStream_t)stream>>>(P, sum_normals, sum_weights, mean_normals);
  return launched("gsr_normal_fusion_mean");
}

int gsr_knn_grid(int n, int k, const float* points, const int* cell_start, const float* grid, int* out_index,
                 float* out_dist, void* stream) {
  if (n <= 0) return 0;
  if (!points || !cell_start || !grid || !out_index || !out_dist) return fail("gsr_knn_grid", "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned nb = blocks(n, 128);
  switch (k) {
    case 1: k_knn_grid<1><<<nb, 128, 0, st>>>(n, points, cell_start, grid, out_index, out_dist); break;
    case 4: k_knn_grid<4><<<nb, 128, 0, st>>>(n, points, cell_start, grid, out_index, out_dist); break;
    case 8: k_knn_grid<8><<<nb, 128, 0, st>>>(n, points, cell_start, grid, out_index, out_dist); break;
    case 10: k_knn_grid<10><<<nb, 128, 0, st>>>(n, points, cell_start, grid, out_index, out_dist); break;
    case 16: k_knn_grid<16><<<nb, 128, 0, st>>>(n, points, cell_start, grid, out_index, out_dist); break;
    default: return fail("gsr_knn_grid", "k must be 1, 4, 8, 10 or 16");
  }
  return launched("gsr_knn_grid");
}

}  // extern "C"
