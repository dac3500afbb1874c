// Marching cubes with the tables of gsr_mc_tables.cuh.  The dense pass over a res^3 grid serves the visual hull
// (gsr_hull.cu) and Shape-as-Points (gsr_sap.cu); the sparse TSDF extraction (gsr_mesh.cu) classifies its own cubes
// and shares the face lookup and the host tail.
//
//   k_mc_dense_count<Corner>          per node g = (i res + j) res + k: the case of the cube whose base it is (all
//                                     three indices < res - 1), that cube's face count, and the crossing edges the
//                                     node owns (+i, +j, +k: bit a), one vertex each.  Every crossing edge of the grid
//                                     lies on a cube.
//   k_mc_dense_emit<Place, REVERSED>  the vertices (Place puts them) and faces, at their scanned offsets; REVERSED
//                                     writes each triangle in the opposite order
//
// Corner: `bool operator()(long long g)`, case bit k set <=> it holds at corner k, so the tables' triangles face the
// side where it holds.  Place: `void operator()(int res, long long g, const int c[3], const long long step[3],
// unsigned mask, float* v)` writes the vertices of the edges node g = c owns (bit a of mask: its +a edge) to v, in
// ascending a, 3 floats each.
#pragma once

#include "gsr_internal.cuh"
#include "../../include/gsr.h"
#include "gsr_mc_tables.cuh"
#include <cub/cub.cuh>

namespace gsr {

// vertex of the crossing on the +a edge of the node (or voxel) go: its first vertex plus its owned edges below a
__device__ __forceinline__ int mc_vertex(const int* __restrict__ vbase, const unsigned char* __restrict__ edges,
                                         long long go, int a) {
  return vbase[go] + __popc(edges[go] & ((1u << a) - 1));
}

template <typename Corner>
__global__ void __launch_bounds__(128) k_mc_dense_count(int res, Corner corner, unsigned char* __restrict__ cube,
                                                        unsigned char* __restrict__ edges, int* __restrict__ fcount,
                                                        int* __restrict__ vcount) {
  const long long N = (long long)res * res * res;
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g > N) return;
  if (g == N) { fcount[N] = 0; vcount[N] = 0; return; }
  const int c[3] = {(int)(g / ((long long)res * res)), (int)((g / res) % res), (int)(g % res)};
  const long long step[3] = {(long long)res * res, res, 1};
  const bool in0 = corner(g);
  unsigned mask = 0;
  for (int a = 0; a < 3; a++)
    if (c[a] + 1 < res && corner(g + step[a]) != in0) mask |= 1u << a;
  unsigned cs = 0;
  const bool full = c[0] + 1 < res && c[1] + 1 < res && c[2] + 1 < res;
  if (full)
    for (int k = 0; k < 8; k++)
      cs |= (unsigned)corner(g + (k & 1) * step[0] + ((k >> 1) & 1) * step[1] + ((k >> 2) & 1) * step[2]) << k;
  cube[g] = (unsigned char)cs;
  edges[g] = (unsigned char)mask;
  fcount[g] = full ? mc_ntri[cs] : 0;
  vcount[g] = __popc(mask);
}

template <typename Place, bool REVERSED>
__global__ void __launch_bounds__(128) k_mc_dense_emit(int res, Place place, const unsigned char* __restrict__ cube,
                                                       const unsigned char* __restrict__ edges,
                                                       const int* __restrict__ vbase, const int* __restrict__ fbase,
                                                       float* __restrict__ verts, long long* __restrict__ faces) {
  const long long N = (long long)res * res * res;
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= N) return;
  const unsigned mask = edges[g], cs = cube[g];
  const int nt = mc_ntri[cs];
  if (!mask && !nt) return;
  const int c[3] = {(int)(g / ((long long)res * res)), (int)((g / res) % res), (int)(g % res)};
  const long long step[3] = {(long long)res * res, res, 1};
  if (mask) place(res, g, c, step, mask, verts + 3 * (size_t)vbase[g]);
  long long fo = fbase[g];
  for (int t = 0; t < nt; t++, fo++)
    for (int j = 0; j < 3; j++) {
      const int e = mc_tri[cs][3 * t + j], c0 = mc_edge[e][0], a = mc_edge[e][2];
      const long long go = g + (c0 & 1) * step[0] + ((c0 >> 1) & 1) * step[1] + ((c0 >> 2) & 1) * step[2];
      faces[3 * fo + (REVERSED ? 2 - j : j)] = mc_vertex(vbase, edges, go, a);
    }
}

static __global__ void k_mc_totals(const int* __restrict__ vbase, const int* __restrict__ fbase, long long N,
                                   unsigned long long* __restrict__ rb) {
  rb[0] = (unsigned long long)vbase[N];
  rb[1] = (unsigned long long)fbase[N];
}

// ---- the host tail every pass shares: scans -> one blocking read of V and F -> outputs -> emit ----
constexpr int MC_RB = 8;  // read-back words: V, F, then any the entry adds (the TSDF volume's counters)
struct McScan {
  int* fbase;              // [N + 1] face count of each cube (entry N: 0), scanned in place into its first face
  int* vbase;              // [N + 1] vertex count of each node, scanned in place into its first vertex
  unsigned long long* rb;  // [MC_RB] device side of the read-back
  char* tmp;
  size_t tmp_bytes;
};
inline void take(char*& p, McScan& s, long long N, cudaStream_t st) {
  s.tmp_bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, s.tmp_bytes, (int*)nullptr, (int)(N + 1), st);
  take(p, s.fbase, N + 1);
  take(p, s.vbase, N + 1);
  take(p, s.rb, MC_RB);
  take(p, s.tmp, s.tmp_bytes);
}
// after the count kernels: both scans, and V, F into s.rb[0], s.rb[1]
inline void mc_scan(const McScan& s, long long N, cudaStream_t st) {
  size_t tmp_bytes = s.tmp_bytes;
  cub::DeviceScan::ExclusiveSum(s.tmp, tmp_bytes, s.fbase, (int)(N + 1), st);
  cub::DeviceScan::ExclusiveSum(s.tmp, tmp_bytes, s.vbase, (int)(N + 1), st);
  k_mc_totals<<<1, 1, 0, st>>>(s.vbase, s.fbase, N, s.rb);
}
// *n_faces = F and, unless V = F = 0, the outputs.  -> 1 allocated, 0 no mesh (nothing allocated), -1 error set
inline int mc_outputs(const char* fn, long long V, long long F, int64_t* n_faces, gsr_alloc_fn vertex_alloc,
                      void* vertex_user, gsr_alloc_fn face_alloc, void* face_user, float*& verts, long long*& faces) {
  *n_faces = F;
  if (V == 0 && F == 0) return 0;
  verts = reinterpret_cast<float*>(vertex_alloc(vertex_user, (size_t)V * 12));
  faces = reinterpret_cast<long long*>(face_alloc(face_user, (size_t)F * 24));
  if (!verts || !faces) return fail(fn, "output allocation failed");
  return 1;
}

// The dense pass: scratch, counts, scans, the read-back, outputs, emit.  Checks no argument (the entry has).
// -> V (0 when there is no mesh), or -1 with the entry's error set.
template <bool REVERSED, typename Corner, typename Place>
int64_t mc_dense(const char* fn, int res, Corner corner, Place place, gsr_alloc_fn scratch_alloc, void* scratch_user,
                 gsr_alloc_fn vertex_alloc, void* vertex_user, gsr_alloc_fn face_alloc, void* face_user,
                 int64_t* n_faces, cudaStream_t st) {
  const long long N = (long long)res * res * res;
  unsigned char *cube, *edges;
  McScan s;
  if (!carve_scratch(fn, scratch_alloc, scratch_user, [&](char*& p) {
        take(p, cube, N);
        take(p, edges, N);
        take(p, s, N, st);
      }))
    return -1;
  k_mc_dense_count<<<blocks(N + 1, 128), 128, 0, st>>>(res, corner, cube, edges, s.fbase, s.vbase);
  mc_scan(s, N, st);
  unsigned long long rb[2];
  if (read_back(fn, s.rb, rb, 2, st)) return -1;
  const long long V = (long long)rb[0];
  float* verts;
  long long* faces;
  const int out = mc_outputs(fn, V, (long long)rb[1], n_faces, vertex_alloc, vertex_user, face_alloc, face_user, verts,
                             faces);
  if (out <= 0) return out;
  k_mc_dense_emit<Place, REVERSED><<<blocks(N, 128), 128, 0, st>>>(res, place, cube, edges, s.vbase, s.fbase, verts,
                                                                    faces);
  return launched(fn) ? -1 : V;
}

}  // namespace gsr
