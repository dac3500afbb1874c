// Mesh extraction on the device: what gaustudio/scripts/extract_mesh.py:86-186 does after the render, there on the
// host through vdbfusion (VDBVolume.integrate / extract_triangle_mesh, float64 point clouds copied out per view) and
// open3d (cluster_connected_triangles).
//
//   k_tsdf_rays<false>   claim the 8^3 bricks a batch of rays adds samples to (open-addressing table, CAS on the key)
//   k_tsdf_rays<true>    add the samples: fixed-point int64 sums + int32 counts, 64-bit atomics
//   k_mc_cubes           per voxel: marching-cubes case of the cube whose corners are v + {0,1}^3, face count
//   k_mc_edges           per voxel: crossing edges it owns (+x, +y, +z) that an active cube uses, vertex count
//   k_mc_emit            vertices (shared, one per crossing edge) and faces, at their scanned offsets; the scans,
//                        the one read-back, the outputs and the face lookup are those of gsr_mc.cuh
//   k_edge_keys / k_union / k_label   triangle components joined by shared edges (union-find)
//
// Claiming and adding are separate launches over the same DDA, so no thread ever waits on a table slot another
// thread is still publishing.  Per-ray arithmetic is float64 with explicit-rounding intrinsics (no FMA contraction)
// and the samples are summed as integers, so the volume does not depend on thread or view order and equals a float64
// numpy restatement (oracle/tsdf_oracle.py) bit for bit.
#include "gsr_internal.cuh"
#include "../../include/gsr.h"
#include "gsr_mc.cuh"
#include <cmath>
#include <string>

namespace gsr {
namespace {

constexpr int BRICK_VOX = 512;                         // 8^3 voxels, local index (z*8 + y)*8 + x
constexpr unsigned long long EMPTY_KEY = ~0ULL;
constexpr long long KEY_OFF = 1LL << 20;               // brick coordinate c is stored as c + 2^20 in 21 bits
constexpr long long MAX_VOXEL = 8 * KEY_OFF;           // |voxel index| < 2^23 on every axis
constexpr double QSCALE = 1048576.0;                   // a sample s is accumulated as rint(s * 2^20 / trunc)
constexpr long long MAX_CAPACITY = 1LL << 18;          // keeps every per-voxel count of the extraction in int32

struct TsdfHeader {            // first 256 B of the state buffer
  unsigned long long n_bricks; // bricks claimed; more than the capacity means the pool ran out
  unsigned long long dropped;  // claims that found no table slot
  unsigned long long far;      // samples outside the addressable voxel range
  double voxel_size, trunc;
};

struct TsdfView {
  TsdfHeader* hdr;
  unsigned long long* table_keys;  // [T] brick key per slot, EMPTY_KEY when free
  int* table_brick;                // [T] brick index of the slot (-1: claimed beyond the capacity)
  unsigned long long* brick_keys;  // [cap] key of each brick index (EMPTY_KEY when unused)
  long long* sums;                 // [cap][512] fixed-point sample sums
  int* weights;                    // [cap][512] sample counts
  long long cap;
  unsigned long long tmask;        // T - 1
};

// The table holds up to 4x the brick pool (at least 64 Ki keys), so a pool that runs out still counts the distinct
// bricks the scene needs and the error can name that number; within the pool the load factor stays <= 1/4.
inline unsigned long long table_size(long long cap) {
  unsigned long long t = 1;
  while (t < 4ULL * (unsigned long long)cap || t < 65536ULL) t <<= 1;
  return t;
}
size_t tsdf_layout(char* base, long long cap, TsdfView* v) {
  const unsigned long long T = table_size(cap);
  size_t off = 256;
  const size_t o_tk = off; off = align256(off + T * 8);
  const size_t o_tb = off; off = align256(off + T * 4);
  const size_t o_bk = off; off = align256(off + (size_t)cap * 8);
  const size_t o_s = off;  off = align256(off + (size_t)cap * BRICK_VOX * 8);
  const size_t o_w = off;  off = align256(off + (size_t)cap * BRICK_VOX * 4);
  if (v) {
    v->hdr = reinterpret_cast<TsdfHeader*>(base);
    v->table_keys = reinterpret_cast<unsigned long long*>(base + o_tk);
    v->table_brick = reinterpret_cast<int*>(base + o_tb);
    v->brick_keys = reinterpret_cast<unsigned long long*>(base + o_bk);
    v->sums = reinterpret_cast<long long*>(base + o_s);
    v->weights = reinterpret_cast<int*>(base + o_w);
    v->cap = cap;
    v->tmask = T - 1;
  }
  return off;
}

__host__ __device__ __forceinline__ unsigned long long brick_key(long long bx, long long by, long long bz) {
  return ((unsigned long long)(bz + KEY_OFF) << 42) | ((unsigned long long)(by + KEY_OFF) << 21) |
         (unsigned long long)(bx + KEY_OFF);
}
__device__ __forceinline__ long long key_coord(unsigned long long key, int axis) {
  return (long long)((key >> (21 * axis)) & ((1ULL << 21) - 1)) - KEY_OFF;
}
__device__ __forceinline__ unsigned long long slot_of(unsigned long long key, unsigned long long mask) {
  key ^= key >> 33; key *= 0xff51afd7ed558ccdULL; key ^= key >> 33; key *= 0xc4ceb9fe1a85ec53ULL; key ^= key >> 33;
  return key & mask;
}

__device__ void claim_brick(const TsdfView& v, unsigned long long key) {
  unsigned long long s = slot_of(key, v.tmask);
  for (unsigned long long probe = 0; probe <= v.tmask; probe++, s = (s + 1) & v.tmask) {
    const unsigned long long k = v.table_keys[s];
    if (k == key) return;
    if (k != EMPTY_KEY) continue;
    const unsigned long long prev = atomicCAS(v.table_keys + s, EMPTY_KEY, key);
    if (prev == key) return;
    if (prev == EMPTY_KEY) {
      const unsigned long long idx = atomicAdd(&v.hdr->n_bricks, 1ULL);
      v.table_brick[s] = idx < (unsigned long long)v.cap ? (int)idx : -1;
      if (idx < (unsigned long long)v.cap) v.brick_keys[idx] = key;
      return;
    }
  }
  atomicAdd(&v.hdr->dropped, 1ULL);
}

// brick index of `key`, -1 if absent (only valid in a launch after the one that claimed it)
__device__ int find_brick(const TsdfView& v, unsigned long long key) {
  unsigned long long s = slot_of(key, v.tmask);
  for (unsigned long long probe = 0; probe <= v.tmask; probe++, s = (s + 1) & v.tmask) {
    const unsigned long long k = v.table_keys[s];
    if (k == key) return v.table_brick[s];
    if (k == EMPTY_KEY) return -1;
  }
  return -1;
}

// One ray per point: p - o = depth * dir, Amanatides-Woo over t in [max(0, depth - trunc), depth + trunc] (t measured
// from the segment start), both end voxels included; sdf = +-|p - c| at voxel centre c = (i + 0.5) voxel_size, positive
// when dot(c - o, p - c) >= 0.  Samples with sdf > -trunc add min(trunc, sdf).  oracle/tsdf_oracle.py repeats this
// operation by operation; tie-breaking of the DDA: the lowest axis among equal tMax.
template <bool ADD>
__global__ void __launch_bounds__(128) k_tsdf_rays(TsdfView v, long long n, const float* __restrict__ pts,
                                                   const unsigned char* __restrict__ valid, double ox, double oy,
                                                   double oz) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || (valid && !valid[i])) return;
  const double vs = v.hdr->voxel_size, trunc = v.hdr->trunc;
  const double px = pts[3 * i], py = pts[3 * i + 1], pz = pts[3 * i + 2];
  const double dx = __dsub_rn(px, ox), dy = __dsub_rn(py, oy), dz = __dsub_rn(pz, oz);
  const double depth = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
  if (!(depth > 0.0) || !(depth < 1e300)) return;  // a point on the origin, NaN or inf has no ray
  const double ux = __ddiv_rn(dx, depth), uy = __ddiv_rn(dy, depth), uz = __ddiv_rn(dz, depth);
  const double t0 = fmax(0.0, __dsub_rn(depth, trunc)), t1 = __dadd_rn(depth, trunc);
  const double sx = __dadd_rn(ox, __dmul_rn(t0, ux)), sy = __dadd_rn(oy, __dmul_rn(t0, uy)),
               sz = __dadd_rn(oz, __dmul_rn(t0, uz));
  const double ex = __dadd_rn(ox, __dmul_rn(t1, ux)), ey = __dadd_rn(oy, __dmul_rn(t1, uy)),
               ez = __dadd_rn(oz, __dmul_rn(t1, uz));
  const double lim = 1e15;  // beyond this a voxel index is not an integer type any more: the ray is out of range
  if (!(fabs(__ddiv_rn(sx, vs)) < lim && fabs(__ddiv_rn(sy, vs)) < lim && fabs(__ddiv_rn(sz, vs)) < lim &&
        fabs(__ddiv_rn(ex, vs)) < lim && fabs(__ddiv_rn(ey, vs)) < lim && fabs(__ddiv_rn(ez, vs)) < lim)) {
    if (!ADD) atomicAdd(&v.hdr->far, 1ULL);
    return;
  }
  long long c[3] = {(long long)floor(__ddiv_rn(sx, vs)), (long long)floor(__ddiv_rn(sy, vs)),
                    (long long)floor(__ddiv_rn(sz, vs))};
  const long long e[3] = {(long long)floor(__ddiv_rn(ex, vs)), (long long)floor(__ddiv_rn(ey, vs)),
                          (long long)floor(__ddiv_rn(ez, vs))};
  const double s[3] = {sx, sy, sz}, u[3] = {ux, uy, uz};
  int step[3];
  double tmax[3], tdelta[3];
  long long nsteps = 0;
#pragma unroll
  for (int a = 0; a < 3; a++) {
    step[a] = u[a] > 0.0 ? 1 : (u[a] < 0.0 ? -1 : 0);
    tdelta[a] = step[a] ? __ddiv_rn(vs, fabs(u[a])) : INFINITY;
    tmax[a] = step[a] > 0   ? __ddiv_rn(__dsub_rn(__dmul_rn((double)(c[a] + 1), vs), s[a]), u[a])
              : step[a] < 0 ? __ddiv_rn(__dsub_rn(__dmul_rn((double)c[a], vs), s[a]), u[a])
                            : INFINITY;
    nsteps += e[a] > c[a] ? e[a] - c[a] : c[a] - e[a];
  }
  unsigned long long last_key = EMPTY_KEY;
  int brick = -1;
  for (long long k = 0;; k++) {
    const double cx = __dmul_rn(__dadd_rn((double)c[0], 0.5), vs), cy = __dmul_rn(__dadd_rn((double)c[1], 0.5), vs),
                 cz = __dmul_rn(__dadd_rn((double)c[2], 0.5), vs);
    const double qx = __dsub_rn(px, cx), qy = __dsub_rn(py, cy), qz = __dsub_rn(pz, cz);
    const double dist = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(qx, qx), __dmul_rn(qy, qy)), __dmul_rn(qz, qz)));
    const double dot = __dadd_rn(__dadd_rn(__dmul_rn(__dsub_rn(cx, ox), qx), __dmul_rn(__dsub_rn(cy, oy), qy)),
                                 __dmul_rn(__dsub_rn(cz, oz), qz));
    const double sdf = dot >= 0.0 ? dist : -dist;
    if (sdf > -trunc) {
      if (c[0] <= -MAX_VOXEL || c[0] >= MAX_VOXEL || c[1] <= -MAX_VOXEL || c[1] >= MAX_VOXEL ||
          c[2] <= -MAX_VOXEL || c[2] >= MAX_VOXEL) {
        if (!ADD) atomicAdd(&v.hdr->far, 1ULL);
      } else {
        const unsigned long long key = brick_key(c[0] >> 3, c[1] >> 3, c[2] >> 3);
        if (key != last_key) {
          last_key = key;
          if (ADD) brick = find_brick(v, key); else claim_brick(v, key);
        }
        if (ADD && brick >= 0) {
          const long long q = llrint(__ddiv_rn(__dmul_rn(fmin(trunc, sdf), QSCALE), trunc));
          const size_t at = (size_t)brick * BRICK_VOX + (((c[2] & 7) * 8 + (c[1] & 7)) * 8 + (c[0] & 7));
          atomicAdd(reinterpret_cast<unsigned long long*>(v.sums + at), (unsigned long long)q);
          atomicAdd(v.weights + at, 1);
        }
      }
    }
    if (k == nsteps) break;
    const int a = (tmax[0] <= tmax[1] && tmax[0] <= tmax[2]) ? 0 : (tmax[1] <= tmax[2] ? 1 : 2);
    c[a] += step[a];
    tmax[a] = __dadd_rn(tmax[a], tdelta[a]);
  }
}

// ---- extraction: voxels are addressed by g = rank * 512 + local, rank = position of the brick in key order ----
struct MeshCtx {
  TsdfView v;
  const unsigned long long* sorted_keys;  // [cap] brick keys in ascending order (unused slots last)
  const int* rank_of;                      // [cap] brick index -> rank
  const unsigned short* cube;              // [N] case | active << 8
  const unsigned char* edges;              // [N] bit a: owns a vertex on its +a edge
  const int* vbase;                        // [N + 1] first vertex of each voxel
  double min_weight;
};

__device__ __forceinline__ int n_live_bricks(const TsdfView& v) {
  const unsigned long long n = v.hdr->n_bricks;
  return (int)(n < (unsigned long long)v.cap ? n : (unsigned long long)v.cap);
}

// g of voxel (x, y, z) or -1 if its brick does not exist
__device__ long long voxel_g(const MeshCtx& m, long long x, long long y, long long z) {
  if (x <= -MAX_VOXEL || x >= MAX_VOXEL || y <= -MAX_VOXEL || y >= MAX_VOXEL || z <= -MAX_VOXEL || z >= MAX_VOXEL)
    return -1;
  const int b = find_brick(m.v, brick_key(x >> 3, y >> 3, z >> 3));
  if (b < 0) return -1;
  return (long long)m.rank_of[b] * BRICK_VOX + (((z & 7) * 8 + (y & 7)) * 8 + (x & 7));
}
// weight and mean sample (in units of trunc / 2^20) of voxel (x, y, z); weight 0 when unobserved
__device__ int voxel_value(const MeshCtx& m, long long x, long long y, long long z, double& f) {
  const int b = (x <= -MAX_VOXEL || x >= MAX_VOXEL || y <= -MAX_VOXEL || y >= MAX_VOXEL || z <= -MAX_VOXEL ||
                 z >= MAX_VOXEL) ? -1 : find_brick(m.v, brick_key(x >> 3, y >> 3, z >> 3));
  f = 0.0;
  if (b < 0) return 0;
  const size_t at = (size_t)b * BRICK_VOX + (((z & 7) * 8 + (y & 7)) * 8 + (x & 7));
  const int w = m.v.weights[at];
  if (w > 0) f = __ddiv_rn((double)m.v.sums[at], (double)w);
  return w;
}
__device__ __forceinline__ void voxel_of(const MeshCtx& m, long long g, long long& x, long long& y, long long& z) {
  const unsigned long long key = m.sorted_keys[g / BRICK_VOX];
  const int l = (int)(g % BRICK_VOX);
  x = key_coord(key, 0) * 8 + (l & 7); y = key_coord(key, 1) * 8 + ((l >> 3) & 7); z = key_coord(key, 2) * 8 + (l >> 6);
}

__global__ void k_init_header(TsdfHeader* h, double voxel_size, double trunc) {
  h->voxel_size = voxel_size;
  h->trunc = trunc;
}
__global__ void k_iota(int n, int* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = i;
}
__global__ void k_rank(TsdfView v, const int* __restrict__ sorted_idx, int* __restrict__ rank_of) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n_live_bricks(v)) rank_of[sorted_idx[r]] = r;
}

__global__ void __launch_bounds__(128) k_mc_cubes(MeshCtx m, long long N, unsigned short* __restrict__ cube,
                                                  int* __restrict__ fcount) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g > N) return;
  if (g == N || g >= (long long)n_live_bricks(m.v) * BRICK_VOX) {
    if (g < N) cube[g] = 0;
    fcount[g] = 0;
    return;
  }
  long long x, y, z;
  voxel_of(m, g, x, y, z);
  int cs = 0;
  bool active = true;
  for (int k = 0; k < 8 && active; k++) {
    double f;
    const int w = voxel_value(m, x + (k & 1), y + ((k >> 1) & 1), z + ((k >> 2) & 1), f);
    active = w > 0 && (double)w > m.min_weight;
    cs |= (f >= 0.0 ? 1 : 0) << k;
  }
  cube[g] = active ? (unsigned short)(cs | 256) : 0;
  fcount[g] = active ? mc_ntri[cs] : 0;
}

__global__ void __launch_bounds__(128) k_mc_edges(MeshCtx m, long long N, unsigned char* __restrict__ edges,
                                                  int* __restrict__ vcount) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g > N) return;
  if (g == N || g >= (long long)n_live_bricks(m.v) * BRICK_VOX) {
    if (g < N) edges[g] = 0;
    vcount[g] = 0;
    return;
  }
  long long x, y, z;
  voxel_of(m, g, x, y, z);
  double f0;
  const int w0 = voxel_value(m, x, y, z, f0);
  unsigned mask = 0;
  if (w0 > 0 && (double)w0 > m.min_weight) {
    for (int a = 0; a < 3; a++) {
      double f1;
      const int w1 = voxel_value(m, x + (a == 0), y + (a == 1), z + (a == 2), f1);
      if (!(w1 > 0 && (double)w1 > m.min_weight) || (f0 >= 0.0) == (f1 >= 0.0)) continue;
      // the four cubes around the edge have their base at v - o, o in {0,1} on the two other axes
      const int u = (a + 1) % 3, w = (a + 2) % 3;
      bool used = false;
      for (int o = 0; o < 4 && !used; o++) {
        long long b[3] = {x, y, z};
        b[u] -= o & 1; b[w] -= o >> 1;
        const long long gc = voxel_g(m, b[0], b[1], b[2]);
        used = gc >= 0 && (m.cube[gc] & 256);
      }
      if (used) mask |= 1u << a;
    }
  }
  edges[g] = (unsigned char)mask;
  vcount[g] = __popc(mask);
}

__global__ void __launch_bounds__(128) k_mc_emit(MeshCtx m, long long N, const int* __restrict__ fbase,
                                                 float* __restrict__ verts, long long* __restrict__ faces) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= N || g >= (long long)n_live_bricks(m.v) * BRICK_VOX) return;
  const unsigned mask = m.edges[g];
  const unsigned cs = m.cube[g];
  if (!mask && !(cs & 256)) return;
  long long x, y, z;
  voxel_of(m, g, x, y, z);
  const double vs = m.v.hdr->voxel_size;
  if (mask) {
    double f0;
    voxel_value(m, x, y, z, f0);
    const long long base[3] = {x, y, z};
    int vid = m.vbase[g];
    for (int a = 0; a < 3; a++) {
      if (!((mask >> a) & 1)) continue;
      double f1;
      voxel_value(m, x + (a == 0), y + (a == 1), z + (a == 2), f1);
      const double t = __ddiv_rn(f0, __dsub_rn(f0, f1));
      for (int k = 0; k < 3; k++) {
        const double c = __dmul_rn(__dadd_rn((double)base[k], 0.5), vs);
        verts[3 * (size_t)vid + k] = __double2float_rn(k == a ? __dadd_rn(c, __dmul_rn(t, vs)) : c);
      }
      vid++;
    }
  }
  if (cs & 256) {
    const int c = cs & 255, nt = mc_ntri[c];
    long long fo = fbase[g];
    for (int t = 0; t < nt; t++, fo++)
      for (int j = 0; j < 3; j++) {
        const int e = mc_tri[c][3 * t + j], c0 = mc_edge[e][0], a = mc_edge[e][2];
        const long long go = voxel_g(m, x + (c0 & 1), y + ((c0 >> 1) & 1), z + ((c0 >> 2) & 1));
        faces[3 * fo + j] = mc_vertex(m.vbase, m.edges, go, a);
      }
  }
}

__global__ void k_export(TsdfView v, const unsigned long long* __restrict__ sorted_keys,
                         const int* __restrict__ sorted_idx, long long* __restrict__ keys, long long* __restrict__ sums,
                         int* __restrict__ weights) {
  const int r = blockIdx.x;
  if (r >= n_live_bricks(v)) return;
  const size_t src = (size_t)sorted_idx[r] * BRICK_VOX, dst = (size_t)r * BRICK_VOX;
  if (threadIdx.x == 0 && keys) keys[r] = (long long)sorted_keys[r];
  for (int l = threadIdx.x; l < BRICK_VOX; l += blockDim.x) {
    if (sums) sums[dst + l] = v.sums[src + l];
    if (weights) weights[dst + l] = v.weights[src + l];
  }
}

// ---- triangle components: faces sharing an edge (open3d cluster_connected_triangles) ----
__global__ void k_edge_keys(long long F, const long long* __restrict__ faces, long long V,
                            unsigned long long* __restrict__ keys, int* __restrict__ vals) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3 * F) return;
  const long long f = i / 3, j = i % 3;
  const long long a = faces[3 * f + j], b = faces[3 * f + (j + 1) % 3];
  keys[i] = (unsigned long long)(a < b ? a : b) * (unsigned long long)V + (unsigned long long)(a < b ? b : a);
  vals[i] = (int)f;
}
__device__ int uf_find(volatile int* parent, int x) {
  while (true) {
    const int p = parent[x];
    if (p == x) return x;
    const int gp = parent[p];
    if (gp != p) parent[x] = gp;  // path halving: gp is an ancestor of x whatever happened meanwhile
    x = p;
  }
}
// links the larger root under the smaller one, so every component ends with its smallest face index as the root
__global__ void k_union(long long n, const unsigned long long* __restrict__ keys, const int* __restrict__ vals,
                        int* parent) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0 || i >= n || keys[i] != keys[i - 1]) return;
  int a = vals[i], b = vals[i - 1];
  while (true) {
    a = uf_find(parent, a); b = uf_find(parent, b);
    if (a == b) return;
    if (a < b) { const int t = a; a = b; b = t; }
    if (atomicCAS(parent + a, a, b) == a) return;
  }
}
__global__ void k_label(long long F, int* parent, long long* __restrict__ labels) {
  const long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (f < F) labels[f] = uf_find(parent, (int)f);
}

bool cap_ok(const char* fn, long long cap) {
  if (cap >= 1 && cap <= MAX_CAPACITY) return true;
  fail(fn, "capacity_bricks must be in 1..262144");
  return false;
}

// Sorts the bricks by key into scratch; `rest(p)` takes the caller's arrays from the same block, after the sort's own
struct SortedBricks {
  unsigned long long* keys;
  int* idx;
};
template <typename Rest>
bool sort_bricks(const char* fn, const TsdfView& v, gsr_alloc_fn alloc, void* user, Rest rest, SortedBricks& out,
                 cudaStream_t st) {
  const int cap = (int)v.cap;
  size_t sort_tmp = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (const unsigned long long*)nullptr,
                                  (unsigned long long*)nullptr, (const int*)nullptr, (int*)nullptr, cap, 0, 64, st);
  int* iota;
  char* tmp;
  if (!carve_scratch(fn, alloc, user, [&](char*& p) {
        take(p, out.keys, cap);
        take(p, iota, cap);
        take(p, out.idx, cap);
        take(p, tmp, sort_tmp);
        rest(p);
      }))
    return false;
  k_iota<<<blocks(cap, 256), 256, 0, st>>>(cap, iota);
  cub::DeviceRadixSort::SortPairs(tmp, sort_tmp, (const unsigned long long*)v.brick_keys, out.keys, (const int*)iota,
                                  out.idx, cap, 0, 64, st);
  return launched(fn) == 0;
}

// rb: the header's n_bricks, dropped, far
bool volume_ok(const char* fn, const unsigned long long* rb, long long cap) {
  if (rb[0] > (unsigned long long)cap || rb[1]) {
    fail(fn, (rb[1] ? "the TSDF volume needs more than " : "the TSDF volume needs ") + std::to_string(rb[0]) +
                 " bricks but its capacity is " + std::to_string(cap) + " (create it with a larger capacity_bricks)");
    return false;
  }
  if (rb[2]) {
    fail(fn, std::to_string(rb[2]) + " samples or rays fell outside the addressable range (|voxel index| < 2^23)");
    return false;
  }
  return true;
}

}  // namespace
}  // namespace gsr

using namespace gsr;

extern "C" {

size_t gsr_tsdf_bytes(int64_t capacity_bricks) {
  if (capacity_bricks < 1 || capacity_bricks > MAX_CAPACITY) return 0;
  return tsdf_layout(nullptr, capacity_bricks, nullptr);
}

int gsr_tsdf_init(void* state, int64_t capacity_bricks, double voxel_size, double sdf_trunc, void* stream) {
  const char* fn = "gsr_tsdf_init";
  if (!state) return fail(fn, "state is required");
  if (!cap_ok(fn, capacity_bricks)) return -1;
  if (!(voxel_size > 0.0 && voxel_size < 1e30 && sdf_trunc > 0.0 && sdf_trunc < 1e30))
    return fail(fn, "voxel_size and sdf_trunc must be positive and finite");
  cudaStream_t st = (cudaStream_t)stream;
  TsdfView v;
  char* base = static_cast<char*>(state);
  const size_t bytes = tsdf_layout(base, capacity_bricks, &v);
  const size_t keys_end = reinterpret_cast<char*>(v.sums) - base;
  cudaMemsetAsync(base, 0, 256, st);
  cudaMemsetAsync(base + 256, 0xff, keys_end - 256, st);  // table keys, slot bricks, brick keys: all "empty"
  cudaMemsetAsync(v.sums, 0, bytes - keys_end, st);
  k_init_header<<<1, 1, 0, st>>>(v.hdr, voxel_size, sdf_trunc);
  return launched(fn);
}

int gsr_tsdf_integrate(void* state, int64_t capacity_bricks, int64_t n, const float* points,
                       const unsigned char* valid, double origin_x, double origin_y, double origin_z, void* stream) {
  const char* fn = "gsr_tsdf_integrate";
  if (!state) return fail(fn, "state is required");
  if (!cap_ok(fn, capacity_bricks)) return -1;
  if (n < 0) return fail(fn, "n must be >= 0");
  if (n > 0 && !points) return fail(fn, "points is required");
  if (!(std::fabs(origin_x) < 1e300 && std::fabs(origin_y) < 1e300 && std::fabs(origin_z) < 1e300))
    return fail(fn, "origin must be finite");
  if (n == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  TsdfView v;
  tsdf_layout(static_cast<char*>(state), capacity_bricks, &v);
  k_tsdf_rays<false><<<blocks(n, 128), 128, 0, st>>>(v, n, points, valid, origin_x, origin_y, origin_z);
  k_tsdf_rays<true><<<blocks(n, 128), 128, 0, st>>>(v, n, points, valid, origin_x, origin_y, origin_z);
  return launched(fn);
}

int64_t gsr_tsdf_extract(void* state, int64_t capacity_bricks, double min_weight, gsr_alloc_fn scratch_alloc,
                         void* scratch_user, gsr_alloc_fn vertex_alloc, void* vertex_user, gsr_alloc_fn face_alloc,
                         void* face_user, int64_t* n_faces, void* stream) {
  const char* fn = "gsr_tsdf_extract";
  if (!state) return fail(fn, "state is required");
  if (!cap_ok(fn, capacity_bricks)) return -1;
  if (!(min_weight >= 0.0)) return fail(fn, "min_weight must be >= 0");
  if (!scratch_alloc || !vertex_alloc || !face_alloc || !n_faces) return fail(fn, "allocators and n_faces are required");
  cudaStream_t st = (cudaStream_t)stream;
  TsdfView v;
  tsdf_layout(static_cast<char*>(state), capacity_bricks, &v);
  const long long N = capacity_bricks * BRICK_VOX;
  int* rank_of;
  unsigned short* cube;
  unsigned char* edges;
  McScan sc;
  SortedBricks sb;
  if (!sort_bricks(fn, v, scratch_alloc, scratch_user, [&](char*& p) {
        take(p, rank_of, capacity_bricks);
        take(p, cube, N);
        take(p, edges, N);
        take(p, sc, N, st);
      }, sb, st))
    return -1;
  MeshCtx m;
  m.v = v;
  m.sorted_keys = sb.keys;
  m.rank_of = rank_of; m.cube = cube; m.edges = edges; m.vbase = sc.vbase; m.min_weight = min_weight;
  k_rank<<<blocks(capacity_bricks, 256), 256, 0, st>>>(v, sb.idx, rank_of);
  k_mc_cubes<<<blocks(N + 1, 128), 128, 0, st>>>(m, N, cube, sc.fbase);
  k_mc_edges<<<blocks(N + 1, 128), 128, 0, st>>>(m, N, edges, sc.vbase);
  mc_scan(sc, N, st);
  // the volume's counters ride along in the same read-back: its refusals come before any output is allocated
  cudaMemcpyAsync(sc.rb + 2, &v.hdr->n_bricks, 3 * sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st);
  unsigned long long rb[5];
  if (read_back(fn, sc.rb, rb, 5, st)) return -1;
  if (!volume_ok(fn, rb + 2, capacity_bricks)) return -1;
  const long long V = (long long)rb[0];
  float* verts;
  long long* faces;
  const int out = mc_outputs(fn, V, (long long)rb[1], n_faces, vertex_alloc, vertex_user, face_alloc, face_user, verts,
                             faces);
  if (out <= 0) return out;
  k_mc_emit<<<blocks(N, 128), 128, 0, st>>>(m, N, sc.fbase, verts, faces);
  return launched(fn) ? -1 : V;
}

int64_t gsr_tsdf_export(void* state, int64_t capacity_bricks, gsr_alloc_fn scratch_alloc, void* scratch_user,
                        int64_t* brick_keys, int64_t* sums, int* weights, void* stream) {
  const char* fn = "gsr_tsdf_export";
  if (!state) return fail(fn, "state is required");
  if (!cap_ok(fn, capacity_bricks)) return -1;
  if (!scratch_alloc) return fail(fn, "scratch_alloc is required");
  cudaStream_t st = (cudaStream_t)stream;
  TsdfView v;
  tsdf_layout(static_cast<char*>(state), capacity_bricks, &v);
  SortedBricks sb;
  if (!sort_bricks(fn, v, scratch_alloc, scratch_user, [](char*&) {}, sb, st)) return -1;
  unsigned long long rb[3];
  if (read_back(fn, &v.hdr->n_bricks, rb, 3, st)) return -1;
  if (!volume_ok(fn, rb, capacity_bricks)) return -1;
  const long long n = (long long)rb[0];
  if (n > 0 && (brick_keys || sums || weights))
    k_export<<<(unsigned)n, 256, 0, st>>>(v, sb.keys, sb.idx, reinterpret_cast<long long*>(brick_keys),
                                          reinterpret_cast<long long*>(sums), weights);
  return launched(fn) ? -1 : n;
}

int gsr_mesh_face_components(int64_t n_faces, const int64_t* faces, int64_t n_vertices, gsr_alloc_fn scratch_alloc,
                             void* scratch_user, int64_t* labels, void* stream) {
  const char* fn = "gsr_mesh_face_components";
  if (n_faces < 0 || n_faces > (1LL << 29)) return fail(fn, "n_faces must be in 0..2^29");
  if (n_vertices < 0 || n_vertices > (1LL << 31)) return fail(fn, "n_vertices must be in 0..2^31");
  if (n_faces == 0) return 0;
  if (!faces || !labels || !scratch_alloc) return fail(fn, "faces, labels and scratch_alloc are required");
  cudaStream_t st = (cudaStream_t)stream;
  const long long F = n_faces, n = 3 * F;
  size_t sort_tmp = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                  (const int*)nullptr, (int*)nullptr, (int)n, 0, 64, st);
  unsigned long long *keys, *keys2;
  int *vals, *vals2, *parent;
  char* tmp;
  if (!carve_scratch(fn, scratch_alloc, scratch_user, [&](char*& p) {
        take(p, keys, n);
        take(p, vals, n);
        take(p, keys2, n);
        take(p, vals2, n);
        take(p, parent, F);
        take(p, tmp, sort_tmp);
      }))
    return -1;
  k_edge_keys<<<blocks(n, 256), 256, 0, st>>>(F, reinterpret_cast<const long long*>(faces), n_vertices, keys, vals);
  cub::DeviceRadixSort::SortPairs(tmp, sort_tmp, (const unsigned long long*)keys, keys2, (const int*)vals, vals2,
                                  (int)n, 0, 64, st);
  k_iota<<<blocks(F, 256), 256, 0, st>>>((int)F, parent);
  k_union<<<blocks(n, 256), 256, 0, st>>>(n, keys2, vals2, parent);
  k_label<<<blocks(F, 256), 256, 0, st>>>(F, parent, reinterpret_cast<long long*>(labels));
  return launched(fn);
}

}  // extern "C"
