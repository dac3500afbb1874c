// Mesh rendering and texturing on the device: the hard z-buffer (pytorch3d MeshRasterizer with faces_per_pixel=1,
// blur_radius=0) that gaustudio/scripts/render_mesh.py and texture_mesh.py stand on, and the two consumers on top.
//
//   k_mr_vertices    per vertex: float64 projection, 1/256-px snapped screen position, view z, usable or not
//   k_mr_faces       per face: drop rules, exact int64 setup; small faces rasterized in place (one 64-bit atomicMin per
//                    covered sample), large ones get a chunk count
//   (cub scan)       chunk counts -> inclusive ends
//   k_mr_large       persistent CTAs pull 16x16-pixel chunks of the large faces from one device ticket
//   k_mr_resolve     key -> face_id / depth, and the key back to empty (no memset before the next view)
//   k_mr_shade       per pixel: normal map and colour image from face_id
//   k_tex_*          one view of texture_mesh: visible faces, selected faces, vertex colours
//
// Coverage and depth use exact integer edge functions and float64 with explicit rounding, and the z-buffer is an
// atomicMin on (float bits of z) << 32 | face, so the result is a pure function of the inputs: it equals the numpy
// restatement in oracle/mesh_raster_oracle.py bit for bit and never depends on scheduling.
#include "gsr_internal.cuh"
#include "../../include/gsr.h"
#include <cub/cub.cuh>
#include <cmath>

namespace gsr {
namespace {

constexpr unsigned long long EMPTY_KEY = ~0ULL;
constexpr double GUARD = 1048576.0;  // |u|, |v| < 2^20 px: snapped coordinates < 2^28, every edge product < 2^60
constexpr int CHUNK = 16;            // large faces are cut into CHUNK x CHUNK pixel chunks, one per CTA ticket
constexpr int LARGE_THREADS = CHUNK * CHUNK;
// A face whose clipped bounding box holds at most this many samples is rasterized by its own thread in the face pass.
#ifndef GSR_MESH_SMALL_MAX
#define GSR_MESH_SMALL_MAX 64
#endif
constexpr int SMALL_MAX = GSR_MESH_SMALL_MAX;
constexpr int MAX_SIDE = 32768;

struct MeshCam {
  double r[9], t[3];  // world -> camera, row-major R and t
  double fx, fy, cx, cy, znear;
  int W, H;
};

struct __align__(16) VRec {
  int x, y;  // snapped position, 1/256 px
  double z;  // view z, -1 when the vertex is not usable
};

struct RasterHeader {
  unsigned long long ticket;  // next chunk of the large-face pass
};

struct RasterCtx {
  MeshCam cam;
  const float* verts;
  const long long* faces;
  long long V, F;
  unsigned long long* keys;  // [H*W]
  RasterHeader* hdr;
  VRec* vrec;                // [V]
  long long* cnt;            // [F] chunks of a large face, 0 otherwise
  long long* ends;           // [F] inclusive scan of cnt
};

struct RasterLayout {
  size_t keys, hdr, vrec, cnt, ends, tmp, tmp_bytes, total;
};
RasterLayout raster_layout(long long V, long long F, int W, int H) {
  RasterLayout L;
  L.tmp_bytes = 0;
  if (F > 0)
    cub::DeviceScan::InclusiveSum(nullptr, L.tmp_bytes, (const long long*)nullptr, (long long*)nullptr, (int)F);
  L.keys = 0;
  L.hdr = align256((size_t)W * H * 8);
  L.vrec = L.hdr + 256;
  L.cnt = L.vrec + align256((size_t)V * sizeof(VRec));
  L.ends = L.cnt + align256((size_t)F * 8);
  L.tmp = L.ends + align256((size_t)F * 8);
  L.total = L.tmp + align256(L.tmp_bytes);
  return L;
}

// p = R x + t, u = fx px / pz + cx, v = fy py / pz + cy: float64, this order, no contraction
__device__ __forceinline__ void project(const MeshCam& c, const float* __restrict__ v, double& u, double& w,
                                        double& pz) {
  const double x = v[0], y = v[1], z = v[2];
  const double px = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(c.r[0], x), __dmul_rn(c.r[1], y)), __dmul_rn(c.r[2], z)), c.t[0]);
  const double py = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(c.r[3], x), __dmul_rn(c.r[4], y)), __dmul_rn(c.r[5], z)), c.t[1]);
  pz = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(c.r[6], x), __dmul_rn(c.r[7], y)), __dmul_rn(c.r[8], z)), c.t[2]);
  u = __dadd_rn(__ddiv_rn(__dmul_rn(c.fx, px), pz), c.cx);
  w = __dadd_rn(__ddiv_rn(__dmul_rn(c.fy, py), pz), c.cy);
}

__device__ __forceinline__ VRec vertex_record(const MeshCam& c, const float* __restrict__ verts, long long i) {
  double u, w, pz;
  project(c, verts + 3 * i, u, w, pz);
  VRec r;
  const bool ok = pz > c.znear && fabs(u) < GUARD && fabs(w) < GUARD;
  r.x = ok ? (int)llrint(__dmul_rn(256.0, u)) : 0;
  r.y = ok ? (int)llrint(__dmul_rn(256.0, w)) : 0;
  r.z = ok ? pz : -1.0;
  return r;
}

// Triangle setup: oriented edge functions e_i(p) = ex_i * (py - ay_i) - ey_i * (px - ax_i) (edge i is opposite vertex
// i), positive inside; |A| the doubled area; tl_i whether edge i is a top-left edge (y down).
struct Tri {
  long long ax[3], ay[3], ex[3], ey[3];
  long long A;  // |doubled area| > 0
  double z[3];
  bool tl[3];
  int x0, x1, y0, y1;  // clipped bounding box, inclusive (empty when x1 < x0 or y1 < y0)
};

__device__ __forceinline__ long long floor256(long long a) { return a >> 8; }
__device__ __forceinline__ long long ceil256(long long a) { return -((-a) >> 8); }

__device__ bool tri_setup(const VRec& a, const VRec& b, const VRec& c, int W, int H, Tri& t) {
  if (!(a.z > 0.0 && b.z > 0.0 && c.z > 0.0)) return false;
  const long long X[3] = {a.x, b.x, c.x}, Y[3] = {a.y, b.y, c.y};
  const long long A = (X[1] - X[0]) * (Y[2] - Y[0]) - (Y[1] - Y[0]) * (X[2] - X[0]);
  if (A == 0) return false;
  const long long s = A > 0 ? 1 : -1;
#pragma unroll
  for (int i = 0; i < 3; i++) {
    const int j = (i + 1) % 3, k = (i + 2) % 3;  // edge i runs from vertex j to vertex k
    t.ax[i] = X[j]; t.ay[i] = Y[j];
    t.ex[i] = s * (X[k] - X[j]); t.ey[i] = s * (Y[k] - Y[j]);
    t.tl[i] = t.ey[i] < 0 || (t.ey[i] == 0 && t.ex[i] > 0);
  }
  t.A = s * A;
  t.z[0] = a.z; t.z[1] = b.z; t.z[2] = c.z;
  const long long mnx = min(X[0], min(X[1], X[2])), mxx = max(X[0], max(X[1], X[2]));
  const long long mny = min(Y[0], min(Y[1], Y[2])), mxy = max(Y[0], max(Y[1], Y[2]));
  t.x0 = (int)max(0LL, ceil256(mnx)); t.x1 = (int)min((long long)W - 1, floor256(mxx));
  t.y0 = (int)max(0LL, ceil256(mny)); t.y1 = (int)min((long long)H - 1, floor256(mxy));
  return true;
}

__device__ __forceinline__ long long edge_at(const Tri& t, int i, long long px, long long py) {
  return t.ex[i] * (py - t.ay[i]) - t.ey[i] * (px - t.ax[i]);
}
__device__ __forceinline__ bool inside(const Tri& t, const long long e[3]) {
  return (e[0] > 0 || (e[0] == 0 && t.tl[0])) && (e[1] > 0 || (e[1] == 0 && t.tl[1])) &&
         (e[2] > 0 || (e[2] == 0 && t.tl[2]));
}
// perspective-correct view z from the oriented edge values: 1 / (l0/z0 + l1/z1 + l2/z2), l_i = e_i / A
__device__ __forceinline__ float depth_at(const Tri& t, const long long e[3]) {
  const double A = (double)t.A;
  const double s = __dadd_rn(__dadd_rn(__ddiv_rn(__ddiv_rn((double)e[0], A), t.z[0]),
                                       __ddiv_rn(__ddiv_rn((double)e[1], A), t.z[1])),
                             __ddiv_rn(__ddiv_rn((double)e[2], A), t.z[2]));
  return __double2float_rn(__ddiv_rn(1.0, s));
}
__device__ __forceinline__ void deposit(unsigned long long* keys, int W, int px, int py, const Tri& t,
                                        const long long e[3], long long f) {
  const unsigned long long key = ((unsigned long long)__float_as_uint(depth_at(t, e)) << 32) | (unsigned long long)f;
  atomicMin(keys + (size_t)py * W + px, key);
}

// the drawn triangle of face f, or false (bad index, unusable vertex, zero area)
__device__ bool face_tri(const RasterCtx& c, long long f, Tri& t) {
  const long long i0 = c.faces[3 * f], i1 = c.faces[3 * f + 1], i2 = c.faces[3 * f + 2];
  if (i0 < 0 || i0 >= c.V || i1 < 0 || i1 >= c.V || i2 < 0 || i2 >= c.V) return false;
  return tri_setup(c.vrec[i0], c.vrec[i1], c.vrec[i2], c.cam.W, c.cam.H, t);
}

__global__ void __launch_bounds__(256) k_mr_vertices(RasterCtx c) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) c.hdr->ticket = 0;
  if (i < c.V) c.vrec[i] = vertex_record(c.cam, c.verts, i);
}

__global__ void __launch_bounds__(128) k_mr_faces(RasterCtx c) {
  const long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= c.F) return;
  Tri t;
  long long n = 0;
  if (face_tri(c, f, t) && t.x1 >= t.x0 && t.y1 >= t.y0) {
    const int bw = t.x1 - t.x0 + 1, bh = t.y1 - t.y0 + 1;
    if ((long long)bw * bh <= SMALL_MAX) {
      long long row[3];
#pragma unroll
      for (int i = 0; i < 3; i++) row[i] = edge_at(t, i, 256LL * t.x0, 256LL * t.y0);
      for (int py = t.y0; py <= t.y1; py++) {
        long long e[3] = {row[0], row[1], row[2]};
        for (int px = t.x0; px <= t.x1; px++) {
          if (inside(t, e)) deposit(c.keys, c.cam.W, px, py, t, e, f);
#pragma unroll
          for (int i = 0; i < 3; i++) e[i] -= 256 * t.ey[i];
        }
#pragma unroll
        for (int i = 0; i < 3; i++) row[i] += 256 * t.ex[i];
      }
    } else {
      n = (long long)((bw + CHUNK - 1) / CHUNK) * ((bh + CHUNK - 1) / CHUNK);
    }
  }
  c.cnt[f] = n;
}

// Persistent: every CTA takes the next chunk ticket until all chunks of all large faces are done; chunk t belongs to
// the first face whose inclusive end exceeds t.
__global__ void __launch_bounds__(LARGE_THREADS) k_mr_large(RasterCtx c) {
  __shared__ long long s_ticket;
  const long long total = c.ends[c.F - 1];
  const int tx = threadIdx.x % CHUNK, ty = threadIdx.x / CHUNK;
  for (;;) {
    if (threadIdx.x == 0) s_ticket = (long long)atomicAdd(&c.hdr->ticket, 1ULL);
    __syncthreads();
    const long long tk = s_ticket;
    __syncthreads();
    if (tk >= total) return;
    long long lo = 0, hi = c.F - 1;
    while (lo < hi) {
      const long long mid = (lo + hi) >> 1;
      if (c.ends[mid] > tk) hi = mid; else lo = mid + 1;
    }
    const long long f = lo, k = tk - (c.ends[f] - c.cnt[f]);
    Tri t;
    face_tri(c, f, t);  // a face with chunks passed every drop rule in k_mr_faces
    const int ncx = (t.x1 - t.x0 + CHUNK) / CHUNK;
    const int ox = t.x0 + (int)(k % ncx) * CHUNK, oy = t.y0 + (int)(k / ncx) * CHUNK;
    const int px = ox + tx, py = oy + ty;
    if (px > t.x1 || py > t.y1) continue;
    long long e[3];
#pragma unroll
    for (int i = 0; i < 3; i++)  // the chunk origin's value, stepped to this thread's sample
      e[i] = edge_at(t, i, 256LL * ox, 256LL * oy) + 256LL * ty * t.ex[i] - 256LL * tx * t.ey[i];
    if (inside(t, e)) deposit(c.keys, c.cam.W, px, py, t, e, f);
  }
}

__global__ void __launch_bounds__(256) k_mr_resolve(long long n, unsigned long long* __restrict__ keys,
                                                    int* __restrict__ face_id, float* __restrict__ depth) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const unsigned long long k = keys[p];
  const bool hit = k != EMPTY_KEY;
  face_id[p] = hit ? (int)(unsigned)(k & 0xffffffffULL) : -1;
  depth[p] = hit ? __uint_as_float((unsigned)(k >> 32)) : -1.0f;
  if (hit) keys[p] = EMPTY_KEY;
}

// the three vertex indices of a face_id entry, or false (no face, or an entry that names no valid face)
__device__ __forceinline__ bool face_vertices(const long long* faces, long long F, long long V, int fid, long long v[3]) {
  if (fid < 0 || fid >= F) return false;
#pragma unroll
  for (int j = 0; j < 3; j++) {
    v[j] = faces[3 * (long long)fid + j];
    if (v[j] < 0 || v[j] >= V) return false;
  }
  return true;
}

// perspective-correct barycentric interpolation at pixel p: weights (l_i / z_i) / sum_j (l_j / z_j)
__device__ __forceinline__ float3 interpolate_color(const MeshCam& cam, const float* __restrict__ verts,
                                                 const long long vi[3], const float* __restrict__ vcolors, long long p) {
  Tri t;
  if (!tri_setup(vertex_record(cam, verts, vi[0]), vertex_record(cam, verts, vi[1]), vertex_record(cam, verts, vi[2]),
                 cam.W, cam.H, t))
    return make_float3(0.f, 0.f, 0.f);
  const long long px = 256LL * (p % cam.W), py = 256LL * (p / cam.W);
  const double w0 = __ddiv_rn(__ddiv_rn((double)edge_at(t, 0, px, py), (double)t.A), t.z[0]);
  const double w1 = __ddiv_rn(__ddiv_rn((double)edge_at(t, 1, px, py), (double)t.A), t.z[1]);
  const double w2 = __ddiv_rn(__ddiv_rn((double)edge_at(t, 2, px, py), (double)t.A), t.z[2]);
  const double sum = __dadd_rn(__dadd_rn(w0, w1), w2);
  const double q0 = __ddiv_rn(w0, sum), q1 = __ddiv_rn(w1, sum), q2 = __ddiv_rn(w2, sum);
  const float* c0 = vcolors + 3 * vi[0];
  const float* c1 = vcolors + 3 * vi[1];
  const float* c2 = vcolors + 3 * vi[2];
  float o[3];
#pragma unroll
  for (int k = 0; k < 3; k++)
    o[k] = __double2float_rn(__dadd_rn(__dadd_rn(__dmul_rn(q0, (double)c0[k]), __dmul_rn(q1, (double)c1[k])),
                                       __dmul_rn(q2, (double)c2[k])));
  return make_float3(o[0], o[1], o[2]);
}

__global__ void __launch_bounds__(256, 1) k_mr_shade(MeshCam cam, const float* __restrict__ verts, long long V,
                                                  const long long* __restrict__ faces, long long F,
                                                  const int* __restrict__ face_id, const float* __restrict__ vnormals,
                                                  const float* __restrict__ vcolors, float* __restrict__ normal,
                                                  float* __restrict__ color) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= (long long)cam.W * cam.H) return;
  long long vi[3];
  const bool hit = face_vertices(faces, F, V, face_id[p], vi);
  if (normal) {
    float o[3] = {0.f, 0.f, 0.f};
    if (hit) {
      float s[3];
#pragma unroll
      for (int k = 0; k < 3; k++) s[k] = __fadd_rn(__fadd_rn(vnormals[3 * vi[0] + k], vnormals[3 * vi[1] + k]),
                                                   vnormals[3 * vi[2] + k]);
      const float len = fmaxf(sqrtf(s[0] * s[0] + s[1] * s[1] + s[2] * s[2]), 1e-12f);
      const float n[3] = {s[0] / len, s[1] / len, s[2] / len};
#pragma unroll
      for (int k = 0; k < 3; k++)
        o[k] = (float)cam.r[3 * k] * n[0] + (float)cam.r[3 * k + 1] * n[1] + (float)cam.r[3 * k + 2] * n[2];
    }
#pragma unroll
    for (int k = 0; k < 3; k++) normal[3 * p + k] = o[k];
  }
  if (color) {
    float3 o = make_float3(0.f, 0.f, 0.f);
    if (hit && !vcolors) o = make_float3(1.f, 1.f, 1.f);
    else if (hit) o = interpolate_color(cam, verts, vi, vcolors, p);
    color[3 * p] = o.x; color[3 * p + 1] = o.y; color[3 * p + 2] = o.z;
  }
}

// ---- texture_mesh, one view ----
__global__ void __launch_bounds__(256) k_tex_visible(long long n, const int* __restrict__ face_id, long long F,
                                                     int stamp, int* __restrict__ face_stamp) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const int f = face_id[p];
  if (f >= 0 && f < F) face_stamp[f] = stamp;
}

constexpr double COS_SCALE = 1099511627776.0;  // 2^40: per-view cosine sums are exact int64 fixed point

__global__ void __launch_bounds__(256) k_tex_faces(MeshCam cam, const float* __restrict__ verts, long long V,
                                                   const long long* __restrict__ faces, long long F, int stamp,
                                                   const int* __restrict__ face_stamp, int* __restrict__ vertex_stamp,
                                                   unsigned long long* __restrict__ stats) {
  const long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long vi[3];
  if (f >= F || face_stamp[f] != stamp || !face_vertices(faces, F, V, (int)f, vi)) return;
  double p[3][3];
#pragma unroll
  for (int j = 0; j < 3; j++)
#pragma unroll
    for (int k = 0; k < 3; k++) p[j][k] = verts[3 * vi[j] + k];
  double e1[3], e2[3];
#pragma unroll
  for (int k = 0; k < 3; k++) { e1[k] = __dsub_rn(p[1][k], p[0][k]); e2[k] = __dsub_rn(p[2][k], p[0][k]); }
  const double n0 = __dsub_rn(__dmul_rn(e1[1], e2[2]), __dmul_rn(e1[2], e2[1]));
  const double n1 = __dsub_rn(__dmul_rn(e1[2], e2[0]), __dmul_rn(e1[0], e2[2]));
  const double n2 = __dsub_rn(__dmul_rn(e1[0], e2[1]), __dmul_rn(e1[1], e2[0]));
  const double len = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(n0, n0), __dmul_rn(n1, n1)), __dmul_rn(n2, n2)));
  if (!(len > 0.0)) return;  // no normal: neither counted nor selected
  const double cosv = __ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(n0, cam.r[6]), __dmul_rn(n1, cam.r[7])),
                                          __dmul_rn(n2, cam.r[8])), len);
  atomicAdd(stats, (unsigned long long)llrint(__dmul_rn(cosv, COS_SCALE)));
  atomicAdd(stats + 1, 1ULL);
  if (cosv < -0.05)
#pragma unroll
    for (int j = 0; j < 3; j++) vertex_stamp[vi[j]] = stamp;
}

__global__ void __launch_bounds__(256) k_tex_vertices(MeshCam cam, const float* __restrict__ verts, long long V,
                                                      int stamp, const int* __restrict__ vertex_stamp,
                                                      const float* __restrict__ image, float* __restrict__ vcolors) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= V || vertex_stamp[i] != stamp) return;
  double u, v, pz;
  project(cam, verts + 3 * i, u, v, pz);
  if (!(u >= 0.0 && u <= (double)(cam.W - 1) && v >= 0.0 && v <= (double)(cam.H - 1))) return;  // NaN fails too
  const int x0 = (int)floor(u), y0 = (int)floor(v);
  const int x1 = min(x0 + 1, cam.W - 1), y1 = min(y0 + 1, cam.H - 1);
  const double ax = __dsub_rn(u, (double)x0), ay = __dsub_rn(v, (double)y0);
  const double bx = __dsub_rn(1.0, ax), by = __dsub_rn(1.0, ay);
  const float* r0 = image + (size_t)y0 * cam.W * 3;
  const float* r1 = image + (size_t)y1 * cam.W * 3;
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const double top = __dadd_rn(__dmul_rn(bx, (double)r0[3 * x0 + k]), __dmul_rn(ax, (double)r0[3 * x1 + k]));
    const double bot = __dadd_rn(__dmul_rn(bx, (double)r1[3 * x0 + k]), __dmul_rn(ax, (double)r1[3 * x1 + k]));
    const double val = __dadd_rn(__dmul_rn(by, top), __dmul_rn(ay, bot));
    vcolors[3 * i + k] = __double2float_rn(fmin(fmax(val, 0.0), 1.0));
  }
}

constexpr long long MAX_COUNT = 2147483647LL;

// The checks every entry point shares, in this order: counts, image size, camera.  The message, or nullptr.
const char* common_error(long long V, long long F, int W, int H, const double* camera, double fx, double fy, double cx,
                         double cy) {
  if (V < 0 || V > MAX_COUNT || F < 0 || F > MAX_COUNT) return "n_vertices and n_faces must be in 0..2^31-1";
  if (W < 1 || W > MAX_SIDE || H < 1 || H > MAX_SIDE) return "width and height must be in 1..32768";
  if (!camera) return "camera is required";
  bool finite = std::isfinite(fx) && std::isfinite(fy) && std::isfinite(cx) && std::isfinite(cy);
  for (int i = 0; i < 12; i++) finite = finite && std::isfinite(camera[i]);
  if (!finite) return "camera, fx, fy, cx and cy must be finite";
  return nullptr;
}
MeshCam make_cam(const double* camera, double fx, double fy, double cx, double cy, double znear, int W, int H) {
  MeshCam c;
  for (int i = 0; i < 9; i++) c.r[i] = camera[i];
  for (int i = 0; i < 3; i++) c.t[i] = camera[9 + i];
  c.fx = fx; c.fy = fy; c.cx = cx; c.cy = cy; c.znear = znear; c.W = W; c.H = H;
  return c;
}

// one wave of the persistent large-face kernel: as many CTAs as are resident at once
int large_grid() {
  int dev = 0, sms = 0, per_sm = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_mr_large, LARGE_THREADS, 0);
  return (sms > 0 ? sms : 1) * (per_sm > 0 ? per_sm : 1);
}

}  // namespace
}  // namespace gsr

using namespace gsr;

extern "C" {

size_t gsr_mesh_raster_bytes(int64_t n_vertices, int64_t n_faces, int width, int height) {
  if (n_vertices < 0 || n_vertices > MAX_COUNT || n_faces < 0 || n_faces > MAX_COUNT || width < 1 ||
      width > MAX_SIDE || height < 1 || height > MAX_SIDE)
    return 0;
  return raster_layout(n_vertices, n_faces, width, height).total;
}

int gsr_mesh_rasterize(int64_t n_vertices, const float* vertices, int64_t n_faces, const int64_t* faces,
                       const double* camera, double fx, double fy, double cx, double cy, double znear, int width,
                       int height, void* scratch, size_t scratch_bytes, int* face_id, float* depth, void* stream) {
  const char* fn = "gsr_mesh_rasterize";
  if (const char* e = common_error(n_vertices, n_faces, width, height, camera, fx, fy, cx, cy)) return fail(fn, e);
  if (!(znear >= 0.0 && std::isfinite(znear))) return fail(fn, "znear must be finite and >= 0");
  if ((n_vertices > 0 && !vertices) || (n_faces > 0 && !faces) || !face_id || !depth || !scratch)
    return fail(fn, "vertices, faces, scratch, face_id and depth are required");
  const RasterLayout L = raster_layout(n_vertices, n_faces, width, height);
  if (scratch_bytes < L.total) return fail(fn, "scratch is smaller than gsr_mesh_raster_bytes");
  cudaStream_t st = (cudaStream_t)stream;
  char* s = static_cast<char*>(scratch);
  RasterCtx c;
  c.cam = make_cam(camera, fx, fy, cx, cy, znear, width, height);
  c.verts = vertices;
  c.faces = reinterpret_cast<const long long*>(faces);
  c.V = n_vertices; c.F = n_faces;
  c.keys = reinterpret_cast<unsigned long long*>(s + L.keys);
  c.hdr = reinterpret_cast<RasterHeader*>(s + L.hdr);
  c.vrec = reinterpret_cast<VRec*>(s + L.vrec);
  c.cnt = reinterpret_cast<long long*>(s + L.cnt);
  c.ends = reinterpret_cast<long long*>(s + L.ends);
  k_mr_vertices<<<blocks(n_vertices > 0 ? n_vertices : 1, 256), 256, 0, st>>>(c);
  if (n_faces > 0) {
    k_mr_faces<<<blocks(n_faces, 128), 128, 0, st>>>(c);
    size_t tmp = L.tmp_bytes;
    cub::DeviceScan::InclusiveSum(s + L.tmp, tmp, (const long long*)c.cnt, c.ends, (int)n_faces, st);
    k_mr_large<<<large_grid(), LARGE_THREADS, 0, st>>>(c);
  }
  const long long n = (long long)width * height;
  k_mr_resolve<<<blocks(n, 256), 256, 0, st>>>(n, c.keys, face_id, depth);
  return launched(fn);
}

int gsr_mesh_shade(int64_t n_vertices, const float* vertices, int64_t n_faces, const int64_t* faces,
                   const double* camera, double fx, double fy, double cx, double cy, int width, int height,
                   const int* face_id, const float* vertex_normals, const float* vertex_colors, float* normal,
                   float* color, void* stream) {
  const char* fn = "gsr_mesh_shade";
  if (const char* e = common_error(n_vertices, n_faces, width, height, camera, fx, fy, cx, cy)) return fail(fn, e);
  if (!face_id || (n_faces > 0 && !faces) || (n_vertices > 0 && !vertices))
    return fail(fn, "vertices, faces and face_id are required");
  if (normal && n_vertices > 0 && !vertex_normals) return fail(fn, "a normal map needs vertex_normals");
  if (!normal && !color) return 0;
  const long long n = (long long)width * height;
  k_mr_shade<<<blocks(n, 256), 256, 0, (cudaStream_t)stream>>>(
      make_cam(camera, fx, fy, cx, cy, 0.0, width, height), vertices, n_vertices,
      reinterpret_cast<const long long*>(faces), n_faces, face_id, vertex_normals, vertex_colors, normal, color);
  return launched(fn);
}

int gsr_mesh_texture_view(int64_t n_vertices, const float* vertices, int64_t n_faces, const int64_t* faces,
                          const double* camera, double fx, double fy, double cx, double cy, int width, int height,
                          const int* face_id, const float* image, int view, int* face_stamp, int* vertex_stamp,
                          int64_t* stats, float* vertex_colors, void* stream) {
  const char* fn = "gsr_mesh_texture_view";
  if (const char* e = common_error(n_vertices, n_faces, width, height, camera, fx, fy, cx, cy)) return fail(fn, e);
  if (view < 0 || view >= 2147483647) return fail(fn, "view must be in 0..2^31-2");
  if (!face_id || !image || !face_stamp || !vertex_stamp || !stats || !vertex_colors ||
      (n_faces > 0 && !faces) || (n_vertices > 0 && !vertices))
    return fail(fn, "vertices, faces, face_id, image, face_stamp, vertex_stamp, stats and vertex_colors are required");
  if (n_faces == 0 || n_vertices == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const MeshCam cam = make_cam(camera, fx, fy, cx, cy, 0.0, width, height);
  const long long n = (long long)width * height;
  const long long* f = reinterpret_cast<const long long*>(faces);
  k_tex_visible<<<blocks(n, 256), 256, 0, st>>>(n, face_id, n_faces, view + 1, face_stamp);
  k_tex_faces<<<blocks(n_faces, 256), 256, 0, st>>>(cam, vertices, n_vertices, f, n_faces, view + 1, face_stamp,
                                                     vertex_stamp, reinterpret_cast<unsigned long long*>(stats));
  k_tex_vertices<<<blocks(n_vertices, 256), 256, 0, st>>>(cam, vertices, n_vertices, view + 1, vertex_stamp, image,
                                                          vertex_colors);
  return launched(fn);
}

}  // extern "C"
