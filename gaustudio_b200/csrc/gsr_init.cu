// Gaussian initialization from geometry: what gaustudio/pipelines/initializers/{pcd,mesh}.py do on the host with torch,
// numpy and open3d.  (distCUDA2, the scale of every initializer without one, is MODE_DIST2 of the neighbour search in
// gsr_clean.cu.)
//
//   normal2rotation                    pcd.py:12-37 in float32, the reference's op order, no contraction
//   k_init_n2r                         that function per point (the pcd initializer's rotations)
//   k_init_vn_pairs + radix sort       open3d's compute_vertex_normals: the (vertex, face) pairs sorted stably by
//   k_init_vn_sum                      vertex, then one thread per vertex sums its faces' normals in face order
//   k_init_mesh                        SuGaR placement (mesh.py:74-250): one thread per (face, slot)
//   k_vox_columns / _hits / _emit      voxelisation: candidate cells per triangle column, Akenine-Moller's tribox3
//   + radix sort + run-length encode   the occupied cells in ascending linear index and a CSR of their triangles
//   k_vox_colors                       per voxel, the colour at the closest point of the mesh
#include "gsr_internal.cuh"
#include "../../include/gsr.h"
#include <cub/cub.cuh>
#include <cmath>

namespace gsr {
namespace {

// ---- normal2rotation (pcd.py:12-37): float32 torch ops restated one by one ----
// F.normalize: x / max(||x||, 1e-12)
__device__ __forceinline__ void normalize3(float v[3]) {
  const float nrm = fmaxf(sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(v[0], v[0]), __fmul_rn(v[1], v[1])),
                                         __fmul_rn(v[2], v[2]))), 1e-12f);
  for (int d = 0; d < 3; d++) v[d] = __fdiv_rn(v[d], nrm);
}
__device__ __forceinline__ float sgn(float x) { return x > 0.f ? 1.f : x < 0.f ? -1.f : x; }  // torch.sign (NaN: NaN)

// -> the raw (not normalised) quaternion (w, x, y, z) of R = [R0 | R1 | n]
__device__ __forceinline__ float4 normal2rotation(const float nin[3]) {
  float n[3] = {nin[0], nin[1], nin[2]};
  normalize3(n);
  // R0 = w0 - sum(w0 * n) * n with w0 = (1, 0, 0)
  const float s = __fadd_rn(__fadd_rn(__fmul_rn(1.f, n[0]), __fmul_rn(0.f, n[1])), __fmul_rn(0.f, n[2]));
  float R0[3] = {__fsub_rn(1.f, __fmul_rn(s, n[0])), __fsub_rn(0.f, __fmul_rn(s, n[1])),
                 __fsub_rn(0.f, __fmul_rn(s, n[2]))};
  const float s0 = sgn(R0[0]);
  for (int d = 0; d < 3; d++) R0[d] = __fmul_rn(R0[d], s0);
  normalize3(R0);
  // R1 = cross(n, R0), then R1 *= sign(R1_y) * sign(n_z)
  float R1[3] = {__fsub_rn(__fmul_rn(n[1], R0[2]), __fmul_rn(n[2], R0[1])),
                 __fsub_rn(__fmul_rn(n[2], R0[0]), __fmul_rn(n[0], R0[2])),
                 __fsub_rn(__fmul_rn(n[0], R0[1]), __fmul_rn(n[1], R0[0]))};
  const float s1 = __fmul_rn(sgn(R1[1]), sgn(n[2]));
  for (int d = 0; d < 3; d++) R1[d] = __fmul_rn(R1[d], s1);
  // rotmat2quaternion of R[:, i, :] = (R0_i, R1_i, n_i)
  const float tr = __fadd_rn(__fadd_rn(__fadd_rn(R0[0], R1[1]), n[2]), 1e-6f);
  const float r = __fdiv_rn(sqrtf(__fadd_rn(1.f, tr)), 2.f);
  const float r4 = __fmul_rn(4.f, r);
  return make_float4(r, __fdiv_rn(__fsub_rn(R1[2], n[1]), r4), __fdiv_rn(__fsub_rn(n[0], R0[2]), r4),
                     __fdiv_rn(__fsub_rn(R0[1], R1[0]), r4));
}

// RGB2SH of create_from_attribute, which runs on the model's CUDA device: torch divides a float32 CUDA tensor by a
// host scalar as a product with the reciprocal, formed in double and rounded to float32
constexpr float SH_C0_INV = (float)(1.0 / 0.28209479177387814);
__device__ __forceinline__ float rgb2sh(float c) { return __fmul_rn(__fsub_rn(c, 0.5f), SH_C0_INV); }

__global__ void k_init_n2r(int n, const float* __restrict__ normals, float4* __restrict__ rot) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v[3] = {normals[3 * (size_t)i], normals[3 * (size_t)i + 1], normals[3 * (size_t)i + 2]};
  rot[i] = normal2rotation(v);
}

// ---- open3d's TriangleMesh::ComputeVertexNormals ----
__global__ void k_init_vn_pairs(int nf, const long long* __restrict__ faces, int* __restrict__ key,
                                int* __restrict__ face) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3 * nf) return;
  key[i] = (int)faces[i];
  face[i] = i / 3;
}
__device__ __forceinline__ int lower_bound_int(const int* __restrict__ a, int n, int v) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(a + mid) < v) lo = mid + 1; else hi = mid;
  }
  return lo;
}
// Face normal (v1 - v0) x (v2 - v0) in double (Eigen's cross), summed in ascending face order (the stable sort kept
// it); Eigen's normalize() divides by sqrt of the squared norm and leaves a zero vector as it is.
__global__ void k_init_vn_sum(int nv, int nf, const float* __restrict__ verts, const long long* __restrict__ faces,
                              const int* __restrict__ key, const int* __restrict__ face, float* __restrict__ normals) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nv) return;
  const int a = lower_bound_int(key, 3 * nf, v), e = lower_bound_int(key, 3 * nf, v + 1);
  double s[3] = {0.0, 0.0, 0.0};
  for (int j = a; j < e; j++) {
    const long long f = face[j];
    double p[3][3];
    for (int c = 0; c < 3; c++)
      for (int d = 0; d < 3; d++) p[c][d] = verts[3 * faces[3 * f + c] + d];
    double u[3], w[3];
    for (int d = 0; d < 3; d++) { u[d] = __dsub_rn(p[1][d], p[0][d]); w[d] = __dsub_rn(p[2][d], p[0][d]); }
    s[0] = __dadd_rn(s[0], __dsub_rn(__dmul_rn(u[1], w[2]), __dmul_rn(u[2], w[1])));
    s[1] = __dadd_rn(s[1], __dsub_rn(__dmul_rn(u[2], w[0]), __dmul_rn(u[0], w[2])));
    s[2] = __dadd_rn(s[2], __dsub_rn(__dmul_rn(u[0], w[1]), __dmul_rn(u[1], w[0])));
  }
  const double z = __dadd_rn(__dadd_rn(__dmul_rn(s[0], s[0]), __dmul_rn(s[1], s[1])), __dmul_rn(s[2], s[2]));
  if (z > 0.0) {
    const double l = sqrt(z);
    for (int d = 0; d < 3; d++) s[d] = __ddiv_rn(s[d], l);
  }
  for (int d = 0; d < 3; d++) normals[3 * (size_t)v + d] = (float)s[d];
}

// ---- SuGaR placement (mesh.py:95-141 tables, :212-250 ops) ----
// slots of n in {1, 3, 4, 6}: rows SLOT_BASE[n] .. + n of BARY (float32, as the reference's tensors), radius per n
__constant__ float BARY[14][3] = {
    {1.f / 3, 1.f / 3, 1.f / 3},                                                       // n = 1
    {1.f / 2, 1.f / 4, 1.f / 4}, {1.f / 4, 1.f / 2, 1.f / 4}, {1.f / 4, 1.f / 4, 1.f / 2},  // n = 3
    {1.f / 3, 1.f / 3, 1.f / 3}, {2.f / 3, 1.f / 6, 1.f / 6}, {1.f / 6, 2.f / 3, 1.f / 6},  // n = 4
    {1.f / 6, 1.f / 6, 2.f / 3},
    {2.f / 3, 1.f / 6, 1.f / 6}, {1.f / 6, 2.f / 3, 1.f / 6}, {1.f / 6, 1.f / 6, 2.f / 3},  // n = 6
    {1.f / 6, 5.f / 12, 5.f / 12}, {5.f / 12, 1.f / 6, 5.f / 12}, {5.f / 12, 5.f / 12, 1.f / 6}};
int slot_base(int n) { return n == 1 ? 0 : n == 3 ? 1 : n == 4 ? 4 : n == 6 ? 8 : -1; }
float circle_radius(int n) {  // float64 in the reference, rounded to float32 where it multiplies a float32 tensor
  return (float)(n == 1 ? 1. / 2. / sqrt(3.) : n == 3 ? 1. / 2. / (sqrt(3.) + 1.) : n == 4 ? 1 / (4. * sqrt(3.))
                                                                                         : 1 / (4. + 2. * sqrt(3.)));
}

// sum over the three corners of (value * bary), as torch's (x[:, None] * b[None]).sum(-2)
__device__ __forceinline__ float bary_sum(float a, float b, float c, const float* w) {
  return __fadd_rn(__fadd_rn(__fmul_rn(a, w[0]), __fmul_rn(b, w[1])), __fmul_rn(c, w[2]));
}

__global__ void k_init_mesh(int nf, int n, int base, float radius, const float* __restrict__ verts,
                            const long long* __restrict__ faces, const float* __restrict__ vnormals,
                            const float* __restrict__ colors, float* __restrict__ xyz, float4* __restrict__ rot,
                            float* __restrict__ f_dc, float* __restrict__ scale, float* __restrict__ opacity) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)nf * n) return;
  const long long f = g / n;
  const float* w = BARY[base + (int)(g - f * n)];
  const long long vi[3] = {faces[3 * f], faces[3 * f + 1], faces[3 * f + 2]};
  float p[3][3];
  for (int c = 0; c < 3; c++)
    for (int d = 0; d < 3; d++) p[c][d] = verts[3 * vi[c] + d];
  float nrm[3], col[3];
  for (int d = 0; d < 3; d++) {
    xyz[3 * g + d] = bary_sum(p[0][d], p[1][d], p[2][d], w);
    nrm[d] = bary_sum(vnormals[3 * vi[0] + d], vnormals[3 * vi[1] + d], vnormals[3 * vi[2] + d], w);
    col[d] = colors ? bary_sum(colors[3 * vi[0] + d], colors[3 * vi[1] + d], colors[3 * vi[2] + d], w) : 1.f;
    f_dc[3 * g + d] = rgb2sh(col[d]);
  }
  normalize3(nrm);
  rot[g] = normal2rotation(nrm);
  // edge j = p_j - p_{(j+1) % 3}; its norm in float32; the smallest times the radius, clamped at 0
  float m = INFINITY;
  for (int j = 0; j < 3; j++) {
    float e[3];
    for (int d = 0; d < 3; d++) e[d] = __fsub_rn(p[j][d], p[(j + 1) % 3][d]);
    const float len = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(e[0], e[0]), __fmul_rn(e[1], e[1])), __fmul_rn(e[2], e[2])));
    m = j == 0 ? len : fminf(m, len);
  }
  const float s = fmaxf(__fmul_rn(m, radius), 0.f);
  const float sxy = logf(__fadd_rn(__fmul_rn(s, 2.f), 1e-7f));
  scale[3 * g] = sxy;
  scale[3 * g + 1] = sxy;
  scale[3 * g + 2] = logf(__fadd_rn(__fmul_rn(0.f, 2.f), 1e-7f));
  opacity[g] = INFINITY;  // inverse_sigmoid(1) = log(1 / 0)
}

// ---- voxelisation: open3d's VoxelGrid::CreateFromTriangleMeshWithinBounds ----
// Akenine-Moller's tribox3 in double, in its op order and without contraction; a touch counts as overlap.
__device__ __forceinline__ double dm(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double da(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ds(double a, double b) { return __dsub_rn(a, b); }
// one edge-cross-axis test: p_a = s * (a * va - b * vb) over the two vertices given, radius fa ha + fb hb
__device__ __forceinline__ bool axis_sep(double pa, double pb, double fa, double fb, double h) {
  const double mn = pa < pb ? pa : pb, mx = pa < pb ? pb : pa;
  const double rad = da(dm(fa, h), dm(fb, h));
  return mn > rad || mx < -rad;
}
__device__ bool tribox(const double c[3], double h, const double t[3][3]) {
  double v0[3], v1[3], v2[3], e0[3], e1[3], e2[3];
  for (int d = 0; d < 3; d++) {
    v0[d] = ds(t[0][d], c[d]); v1[d] = ds(t[1][d], c[d]); v2[d] = ds(t[2][d], c[d]);
  }
  for (int d = 0; d < 3; d++) { e0[d] = ds(v1[d], v0[d]); e1[d] = ds(v2[d], v1[d]); e2[d] = ds(v0[d], v2[d]); }
  enum { X = 0, Y = 1, Z = 2 };
  double fex = fabs(e0[X]), fey = fabs(e0[Y]), fez = fabs(e0[Z]);
  // AXISTEST_X01(e0z, e0y, fez, fey), AXISTEST_Y02(e0z, e0x, fez, fex), AXISTEST_Z12(e0y, e0x, fey, fex)
  if (axis_sep(ds(dm(e0[Z], v0[Y]), dm(e0[Y], v0[Z])), ds(dm(e0[Z], v2[Y]), dm(e0[Y], v2[Z])), fez, fey, h)) return false;
  if (axis_sep(da(dm(-e0[Z], v0[X]), dm(e0[X], v0[Z])), da(dm(-e0[Z], v2[X]), dm(e0[X], v2[Z])), fez, fex, h)) return false;
  if (axis_sep(ds(dm(e0[Y], v1[X]), dm(e0[X], v1[Y])), ds(dm(e0[Y], v2[X]), dm(e0[X], v2[Y])), fey, fex, h)) return false;
  fex = fabs(e1[X]); fey = fabs(e1[Y]); fez = fabs(e1[Z]);
  // AXISTEST_X01(e1z, e1y), AXISTEST_Y02(e1z, e1x), AXISTEST_Z0(e1y, e1x)
  if (axis_sep(ds(dm(e1[Z], v0[Y]), dm(e1[Y], v0[Z])), ds(dm(e1[Z], v2[Y]), dm(e1[Y], v2[Z])), fez, fey, h)) return false;
  if (axis_sep(da(dm(-e1[Z], v0[X]), dm(e1[X], v0[Z])), da(dm(-e1[Z], v2[X]), dm(e1[X], v2[Z])), fez, fex, h)) return false;
  if (axis_sep(ds(dm(e1[Y], v0[X]), dm(e1[X], v0[Y])), ds(dm(e1[Y], v1[X]), dm(e1[X], v1[Y])), fey, fex, h)) return false;
  fex = fabs(e2[X]); fey = fabs(e2[Y]); fez = fabs(e2[Z]);
  // AXISTEST_X2(e2z, e2y), AXISTEST_Y1(e2z, e2x), AXISTEST_Z12(e2y, e2x)
  if (axis_sep(ds(dm(e2[Z], v0[Y]), dm(e2[Y], v0[Z])), ds(dm(e2[Z], v1[Y]), dm(e2[Y], v1[Z])), fez, fey, h)) return false;
  if (axis_sep(da(dm(-e2[Z], v0[X]), dm(e2[X], v0[Z])), da(dm(-e2[Z], v1[X]), dm(e2[X], v1[Z])), fez, fex, h)) return false;
  if (axis_sep(ds(dm(e2[Y], v1[X]), dm(e2[X], v1[Y])), ds(dm(e2[Y], v2[X]), dm(e2[X], v2[Y])), fey, fex, h)) return false;
  // bullet 1: the triangle's box against the box
  for (int d = 0; d < 3; d++) {
    const double mn = fmin(fmin(v0[d], v1[d]), v2[d]), mx = fmax(fmax(v0[d], v1[d]), v2[d]);
    if (mn > h || mx < -h) return false;
  }
  // bullet 2: planeBoxOverlap(e0 x e1, v0, h)
  const double nr[3] = {ds(dm(e0[Y], e1[Z]), dm(e0[Z], e1[Y])), ds(dm(e0[Z], e1[X]), dm(e0[X], e1[Z])),
                        ds(dm(e0[X], e1[Y]), dm(e0[Y], e1[X]))};
  double vmin[3], vmax[3];
  for (int d = 0; d < 3; d++) {
    if (nr[d] > 0.0) { vmin[d] = ds(-h, v0[d]); vmax[d] = ds(h, v0[d]); }
    else { vmin[d] = ds(h, v0[d]); vmax[d] = ds(-h, v0[d]); }
  }
  if (da(da(dm(nr[0], vmin[0]), dm(nr[1], vmin[1])), dm(nr[2], vmin[2])) > 0.0) return false;
  return da(da(dm(nr[0], vmax[0]), dm(nr[1], vmax[1])), dm(nr[2], vmax[2])) >= 0.0;
}

// Candidates of a triangle: the columns of its bounding box (grown by one cell) along the two axes other than its
// normal's dominant one, and in each column the cells its plane can reach over the column's footprint, grown by the
// bound on the computed plane's error (Tri::slack) and by one cell (the plane is at most sqrt(2) cells steep per cell
// there, and the rounding of the plane's evaluation and of tribox3 itself is far below a cell).
// The work thus grows with the projected area of the box, not with its volume.
struct Tri {
  double p[3][3];
  int lo[3], hi[3];  // cell range of the grown bounding box, clipped to the grid
  int a, u, w;       // dominant normal axis and the two column axes
  double n[3];
  double slack;      // bound on |n . (q - p0)| / |n_a| over the triangle's points q, from the rounding of n
};
__device__ __forceinline__ int cell_of(double x, double vs, int res) {
  return (int)fmin(fmax(floor(ds(x, -0.5) / vs), -1.0), (double)res);
}
__device__ void load_tri(const double* __restrict__ verts, const long long* __restrict__ faces, long long f, double vs,
                         int res, Tri& T) {
  for (int c = 0; c < 3; c++)
    for (int d = 0; d < 3; d++) T.p[c][d] = verts[3 * faces[3 * f + c] + d];
  for (int d = 0; d < 3; d++) {
    const double mn = fmin(fmin(T.p[0][d], T.p[1][d]), T.p[2][d]), mx = fmax(fmax(T.p[0][d], T.p[1][d]), T.p[2][d]);
    T.lo[d] = max(cell_of(mn, vs, res) - 1, 0);
    T.hi[d] = min(cell_of(mx, vs, res) + 1, res - 1);
  }
  double e[3], g[3];
  for (int d = 0; d < 3; d++) { e[d] = T.p[1][d] - T.p[0][d]; g[d] = T.p[2][d] - T.p[0][d]; }
  T.n[0] = e[1] * g[2] - e[2] * g[1];
  T.n[1] = e[2] * g[0] - e[0] * g[2];
  T.n[2] = e[0] * g[1] - e[1] * g[0];
  T.a = fabs(T.n[0]) >= fabs(T.n[1]) ? (fabs(T.n[0]) >= fabs(T.n[2]) ? 0 : 2) : (fabs(T.n[1]) >= fabs(T.n[2]) ? 1 : 2);
  T.u = (T.a + 1) % 3;
  T.w = (T.a + 2) % 3;
  // A point q = p0 + s e' + t g' of the triangle (s, t >= 0, s + t <= 1, e', g' the exact edges) lies off the computed
  // plane by |n . (q - p0)| <= |n . e'| + |n . g'|.  e, g differ from e', g' by <= u |e'|, u |g'| (u = 2^-53), and n
  // from e x g by <= 4 u |e| |g| per component (two products, one difference; contraction changes only the
  // constant), while e x g is orthogonal to e and g.  So |n . (q - p0)| <= ~10 u |e| |g| (|e| + |g|): 64 u is taken,
  // and divided by |n_a| it bounds the error of the slab's height on axis a.  For a (nearly) collinear triangle n is
  // rounding noise; the slack then covers the whole bounding box.
  const double le = sqrt(e[0] * e[0] + e[1] * e[1] + e[2] * e[2]), lg = sqrt(g[0] * g[0] + g[1] * g[1] + g[2] * g[2]);
  T.slack = 64.0 * 0x1p-53 * le * lg * (le + lg) / fabs(T.n[T.a]);  // +inf when n_a = 0
}
__device__ __forceinline__ long long n_columns(const Tri& T) {
  return (long long)(T.hi[T.u] - T.lo[T.u] + 1) * (T.hi[T.w] - T.lo[T.w] + 1);
}
// the slab [k0, k1] on axis a of column j
__device__ void column(const Tri& T, long long j, double vs, int& iu, int& iw, int& k0, int& k1) {
  const int nu = T.hi[T.u] - T.lo[T.u] + 1;
  iu = T.lo[T.u] + (int)(j % nu);
  iw = T.lo[T.w] + (int)(j / nu);
  k0 = T.lo[T.a];
  k1 = T.hi[T.a];
  if (!(T.slack < 1.0)) return;  // n_a = 0 or pure rounding: the whole box
  double mn = INFINITY, mx = -INFINITY;
  for (int c = 0; c < 4; c++) {
    const double x = -0.5 + (iu + (c & 1)) * vs, y = -0.5 + (iw + (c >> 1)) * vs;
    const double z = T.p[0][T.a] - (T.n[T.u] * (x - T.p[0][T.u]) + T.n[T.w] * (y - T.p[0][T.w])) / T.n[T.a];
    mn = fmin(mn, z);
    mx = fmax(mx, z);
  }
  const int res = 1 << 30;  // no clip here: [k0, k1] clips
  k0 = max(k0, cell_of(mn - T.slack, vs, res) - 1);
  k1 = min(k1, cell_of(mx + T.slack, vs, res) + 1);
}
// linear index (i res + j) res + k of the cell with coordinate c[a] = ka, c[u] = iu, c[w] = iw
__device__ __forceinline__ void cell_box(const Tri& T, int iu, int iw, int ka, double vs, int res, double ctr[3],
                                         unsigned& lin) {
  int c[3];
  c[T.a] = ka; c[T.u] = iu; c[T.w] = iw;
  for (int d = 0; d < 3; d++) ctr[d] = da(da(-0.5, dm((double)c[d], vs)), vs / 2);
  lin = ((unsigned)c[0] * res + c[1]) * res + c[2];
}

__global__ void k_vox_columns(int nf, const double* __restrict__ verts, const long long* __restrict__ faces, double vs,
                              int res, long long* __restrict__ ncol) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > nf) return;
  if (f == nf) { ncol[f] = 0; return; }
  Tri T;
  load_tri(verts, faces, f, vs, res, T);
  ncol[f] = n_columns(T);
}
// thread per column: its triangle is the last f with col_off[f] <= c
__device__ __forceinline__ int column_owner(const long long* __restrict__ off, int nf, long long c) {
  int lo = 0, hi = nf;  // off[lo] <= c < off[hi]
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(off + mid) <= c) lo = mid; else hi = mid;
  }
  return lo;
}
template <bool EMIT>
__global__ void k_vox_hits(int nf, long long ncols, const double* __restrict__ verts, const long long* __restrict__ faces,
                           double vs, int res, const long long* __restrict__ col_off, long long* __restrict__ hits,
                           unsigned* __restrict__ cell, int* __restrict__ tri) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c > ncols) return;
  if (!EMIT && c == ncols) { hits[c] = 0; return; }
  if (c == ncols) return;
  const int f = column_owner(col_off, nf, c);
  Tri T;
  load_tri(verts, faces, f, vs, res, T);
  int iu, iw, k0, k1;
  column(T, c - col_off[f], vs, iu, iw, k0, k1);
  const double h = vs / 2;
  long long out = EMIT ? hits[c] : 0;
  for (int ka = k0; ka <= k1; ka++) {
    double ctr[3];
    unsigned lin;
    cell_box(T, iu, iw, ka, vs, res, ctr, lin);
    if (!tribox(ctr, h, T.p)) continue;
    if (EMIT) { cell[out] = lin; tri[out] = f; }
    out++;
  }
  if (!EMIT) hits[c] = out;
}
__global__ void k_vox_total(const long long* __restrict__ a, long long n, long long* __restrict__ out) { *out = a[n]; }

// ---- closest point of a triangle in double: the squared distance and the barycentrics of the point ----
// squared distance from p to u a + v b + w c
__device__ __forceinline__ double dist_at(const double p[3], const double a[3], const double b[3], const double c[3],
                                          double u, double v, double w) {
  double q2 = 0.0;
  for (int d = 0; d < 3; d++) {
    const double e = ds(p[d], da(da(dm(u, a[d]), dm(v, b[d])), dm(w, c[d])));
    q2 = da(q2, dm(e, e));
  }
  return q2;
}
// Candidates, the first smallest winning: the plane's foot when it falls inside (Ericson's va, vb, vc >= 0 with a
// positive sum, Real-Time Collision Detection 5.1.5), then the clamped projections onto the edges ab, bc, ca (a zero
// edge gives its vertex).  The distance to the closed triangle is the least of these, every candidate is a point of
// the triangle, and every ratio has a positive denominator, so a degenerate face (a zero edge, collinear vertices)
// still gets its exact, finite closest point.
__device__ double closest_bary(const double p[3], const double a[3], const double b[3], const double c[3],
                               double bc[3]) {
  double ab[3], ac[3], ap[3], bp[3], cp[3];
  for (int d = 0; d < 3; d++) {
    ab[d] = ds(b[d], a[d]); ac[d] = ds(c[d], a[d]); ap[d] = ds(p[d], a[d]); bp[d] = ds(p[d], b[d]);
    cp[d] = ds(p[d], c[d]);
  }
  auto dot = [](const double* x, const double* y) { return da(da(dm(x[0], y[0]), dm(x[1], y[1])), dm(x[2], y[2])); };
  const double d1 = dot(ab, ap), d2 = dot(ac, ap), d3 = dot(ab, bp), d4 = dot(ac, bp), d5 = dot(ab, cp),
               d6 = dot(ac, cp);
  const double vc = ds(dm(d1, d4), dm(d3, d2)), vb = ds(dm(d5, d2), dm(d1, d6)), va = ds(dm(d3, d6), dm(d5, d4));
  const double den = da(da(va, vb), vc);
  double best = INFINITY;
  bc[0] = 1.0; bc[1] = 0.0; bc[2] = 0.0;
  if (den > 0.0 && va >= 0.0 && vb >= 0.0 && vc >= 0.0) {
    const double v = __ddiv_rn(vb, den), w = __ddiv_rn(vc, den), u = ds(ds(1.0, v), w);
    best = dist_at(p, a, b, c, u, v, w);
    bc[0] = u; bc[1] = v; bc[2] = w;
  }
  const double* P[3] = {a, b, c};
  for (int s = 0; s < 3; s++) {
    const double *x = P[s], *y = P[(s + 1) % 3];
    double dd[3], px[3];
    for (int d = 0; d < 3; d++) { dd[d] = ds(y[d], x[d]); px[d] = ds(p[d], x[d]); }
    const double L = dot(dd, dd);
    const double t = L > 0.0 ? fmin(fmax(__ddiv_rn(dot(px, dd), L), 0.0), 1.0) : 0.0;
    double cb[3] = {0.0, 0.0, 0.0};
    cb[s] = ds(1.0, t);
    cb[(s + 1) % 3] = t;
    const double dc = dist_at(p, a, b, c, cb[0], cb[1], cb[2]);
    if (dc < best) { best = dc; bc[0] = cb[0]; bc[1] = cb[1]; bc[2] = cb[2]; }
  }
  return best;
}
// the voxel's centre as open3d's VoxelGrid::GetVoxelCenterCoordinate forms it: (idx + 0.5) * voxel_size + origin
__device__ __forceinline__ double voxel_centre(int idx, double vs) { return da(dm(da((double)idx, 0.5), vs), -0.5); }
__device__ __forceinline__ int find_cell(const unsigned* __restrict__ cells, int n, unsigned v) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(cells + mid) < v) lo = mid + 1; else hi = mid;
  }
  return lo < n && cells[lo] == v ? lo : -1;
}
// Some triangle meets the voxel's own box (it is occupied), so the mesh's closest point to the centre lies within
// sqrt(3)/2 cell of it, and every triangle that comes that close meets a box of the 3x3x3 block around the voxel
// (their union holds the ball of radius 1 cell around the centre).  Those boxes are occupied cells with the triangle
// in their lists, so the search over them is exact.
__global__ void k_vox_colors(int ncell, const unsigned* __restrict__ cells, const int* __restrict__ off,
                             const int* __restrict__ tris, int res, double vs, const double* __restrict__ verts,
                             const long long* __restrict__ faces, const float* __restrict__ colors,
                             float* __restrict__ rgb) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ncell) return;
  const unsigned lin = cells[i];
  const int c[3] = {(int)(lin / ((unsigned)res * res)), (int)(lin / res % res), (int)(lin % res)};
  double p[3];
  for (int d = 0; d < 3; d++) p[d] = voxel_centre(c[d], vs);
  // seeded with the first triangle of the voxel's own list, so bt is always a face of the mesh
  int bt = tris[off[i]];
  double bb[3], best;
  {
    double v[3][3];
    for (int a = 0; a < 3; a++)
      for (int d = 0; d < 3; d++) v[a][d] = verts[3 * faces[3 * (long long)bt + a] + d];
    best = closest_bary(p, v[0], v[1], v[2], bb);
  }
  for (int o = 0; o < 27; o++) {
    const int q[3] = {c[0] + o / 9 - 1, c[1] + o / 3 % 3 - 1, c[2] + o % 3 - 1};
    if (q[0] < 0 || q[1] < 0 || q[2] < 0 || q[0] >= res || q[1] >= res || q[2] >= res) continue;
    const int k = find_cell(cells, ncell, ((unsigned)q[0] * res + q[1]) * res + q[2]);
    if (k < 0) continue;
    for (int j = off[k]; j < off[k + 1]; j++) {
      const int t = tris[j];
      double v[3][3], bc[3];
      for (int a = 0; a < 3; a++)
        for (int d = 0; d < 3; d++) v[a][d] = verts[3 * faces[3 * (long long)t + a] + d];
      const double d2 = closest_bary(p, v[0], v[1], v[2], bc);
      if (d2 < best || (d2 == best && t < bt)) {
        best = d2; bt = t;
        for (int d = 0; d < 3; d++) bb[d] = bc[d];
      }
    }
  }
  for (int d = 0; d < 3; d++) {
    double s = 0.0;
    for (int a = 0; a < 3; a++) s = da(s, dm(bb[a], (double)colors[3 * faces[3 * (long long)bt + a] + d]));
    rgb[3 * (size_t)i + d] = (float)s;
  }
}

}  // namespace
}  // namespace gsr

using namespace gsr;

extern "C" {

int gsr_normal2rotation(int64_t n, const float* normals, float* rot, void* stream) {
  const char* fn = "gsr_normal2rotation";
  if (!count_ok(fn, n, "n")) return -1;
  if (!normals || !rot) return fail(fn, "normals and rot are required");
  if (misaligned16(rot)) return fail(fn, "rot must be 16-byte aligned");
  k_init_n2r<<<blocks(n, 256), 256, 0, (cudaStream_t)stream>>>((int)n, normals, reinterpret_cast<float4*>(rot));
  return launched(fn);
}

int gsr_mesh_vertex_normals(int64_t nv, const float* verts, int64_t nf, const int64_t* faces,
                            gsr_alloc_fn scratch_alloc, void* scratch_user, float* normals, void* stream) {
  const char* fn = "gsr_mesh_vertex_normals";
  if (!count_ok(fn, nv, "nv") || !count_ok(fn, nf, "nf")) return -1;
  if (nf > 0x7fffffffLL / 3) return fail(fn, "nf must be below 2^31 / 3");
  if (!verts || !faces || !scratch_alloc || !normals) return fail(fn, "verts, faces, scratch_alloc and normals are required");
  cudaStream_t st = (cudaStream_t)stream;
  const int m = 3 * (int)nf;
  int bits = 1;
  while (bits < 31 && (1ll << bits) < nv) bits++;
  size_t sort_tmp = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (const int*)nullptr, (int*)nullptr, (const int*)nullptr,
                                  (int*)nullptr, m, 0, bits, st);
  int *key, *face, *key2, *face2;
  char* tmp;
  if (!carve_scratch(fn, scratch_alloc, scratch_user, [&](char*& p) {
        take(p, key, m);
        take(p, face, m);
        take(p, key2, m);
        take(p, face2, m);
        take(p, tmp, sort_tmp);
      }))
    return -1;
  const long long* f64 = reinterpret_cast<const long long*>(faces);
  k_init_vn_pairs<<<blocks(m, 256), 256, 0, st>>>((int)nf, f64, key, face);
  cub::DeviceRadixSort::SortPairs(tmp, sort_tmp, (const int*)key, key2, (const int*)face, face2, m, 0, bits, st);
  k_init_vn_sum<<<blocks(nv, 128), 128, 0, st>>>((int)nv, (int)nf, verts, f64, key2, face2, normals);
  return launched(fn);
}

int gsr_mesh_gaussians(int64_t nf, int n, const float* verts, const int64_t* faces, const float* vertex_normals,
                       const float* colors, float* xyz, float* rot, float* f_dc, float* scale, float* opacity,
                       void* stream) {
  const char* fn = "gsr_mesh_gaussians";
  if (!count_ok(fn, nf, "nf")) return -1;
  const int base = slot_base(n);
  if (base < 0) return fail(fn, "n must be 1, 3, 4 or 6");
  if (!verts || !faces || !vertex_normals || !xyz || !rot || !f_dc || !scale || !opacity)
    return fail(fn, "verts, faces, vertex_normals and every output are required");
  if (misaligned16(rot)) return fail(fn, "rot must be 16-byte aligned");
  k_init_mesh<<<blocks(nf * n, 256), 256, 0, (cudaStream_t)stream>>>(
      (int)nf, n, base, circle_radius(n), verts, reinterpret_cast<const long long*>(faces), vertex_normals, colors, xyz,
      reinterpret_cast<float4*>(rot), f_dc, scale, opacity);
  return launched(fn);
}

int64_t gsr_voxelize(int64_t nv, const double* verts, int64_t nf, const int64_t* faces, int res, double voxel_size,
                     gsr_alloc_fn alloc, void* column_user, void* hit_user, void* sort_user, void* out_user,
                     int64_t* n_pairs, void* stream) {
  const char* fn = "gsr_voxelize";
  if (!count_ok(fn, nv, "nv") || !count_ok(fn, nf, "nf")) return -1;
  if (res < 1 || res > 1024) return fail(fn, "res must be in 1..1024");
  if (!(voxel_size > 0.0 && voxel_size < INFINITY)) return fail(fn, "voxel_size must be positive and finite");
  if (!verts || !faces || !alloc || !n_pairs) return fail(fn, "verts, faces, alloc and n_pairs are required");
  cudaStream_t st = (cudaStream_t)stream;
  const int F = (int)nf;
  const long long* f64 = reinterpret_cast<const long long*>(faces);
  long long C = 0, H = 0, U = 0;
  // 1. columns per triangle
  size_t tmp = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tmp, (long long*)nullptr, (long long*)nullptr, F + 1, st);
  long long *col_off, *rb;
  char* tmp1;
  if (!carve_scratch(fn, alloc, column_user, [&](char*& p) {
        take(p, col_off, F + 1);
        take(p, rb, 1);
        take(p, tmp1, tmp);
      }))
    return -1;
  k_vox_columns<<<blocks(F + 1, 256), 256, 0, st>>>(F, verts, f64, voxel_size, res, col_off);
  cub::DeviceScan::ExclusiveSum(tmp1, tmp, col_off, col_off, F + 1, st);
  k_vox_total<<<1, 1, 0, st>>>(col_off, F, rb);
  if (read_back(fn, rb, &C, 1, st)) return -1;
  // 2. overlapping cells per column
  tmp = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tmp, (long long*)nullptr, (long long*)nullptr, C + 1, st);
  long long* hits;
  char* tmp2;
  if (!carve_scratch(fn, alloc, hit_user, [&](char*& p) {
        take(p, hits, C + 1);
        take(p, tmp2, tmp);
      }))
    return -1;
  k_vox_hits<false><<<blocks(C + 1, 128), 128, 0, st>>>(F, C, verts, f64, voxel_size, res, col_off, hits, nullptr,
                                                         nullptr);
  cub::DeviceScan::ExclusiveSum(tmp2, tmp, hits, hits, C + 1, st);
  k_vox_total<<<1, 1, 0, st>>>(hits, C, rb);
  if (read_back(fn, rb, &H, 1, st)) return -1;
  *n_pairs = H;
  if (H == 0) return 0;
  if (H > 0x7fffffffLL) return fail(fn, "more than 2^31-1 (cell, triangle) pairs");
  // 3. the pairs, sorted by cell (stable: triangles stay ascending), and the runs of equal cells
  int bits = 1;
  while (bits < 32 && (1ull << bits) < (unsigned long long)res * res * res) bits++;
  size_t sort_tmp = 0, rle_tmp = 0, scan_tmp = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (const unsigned*)nullptr, (unsigned*)nullptr, (const int*)nullptr,
                                  (int*)nullptr, (int)H, 0, bits, st);
  cub::DeviceRunLengthEncode::Encode(nullptr, rle_tmp, (const unsigned*)nullptr, (unsigned*)nullptr, (int*)nullptr,
                                     (long long*)nullptr, (int)H, st);
  cub::DeviceScan::ExclusiveSum(nullptr, scan_tmp, (int*)nullptr, (int*)nullptr, (int)H + 1, st);
  unsigned *cell, *cell2, *ucell;
  int *tri, *tri2, *cnt;
  long long* nrun;
  char* tmp3;
  if (!carve_scratch(fn, alloc, sort_user, [&](char*& p) {
        take(p, cell, H + 1);
        take(p, cell2, H + 1);
        take(p, ucell, H + 1);
        take(p, tri, H + 1);
        take(p, tri2, H + 1);
        take(p, cnt, H + 1);
        take(p, nrun, 1);
        take(p, tmp3, std::max(sort_tmp, std::max(rle_tmp, scan_tmp)));
      }))
    return -1;
  k_vox_hits<true><<<blocks(C + 1, 128), 128, 0, st>>>(F, C, verts, f64, voxel_size, res, col_off, hits, cell, tri);
  cub::DeviceRadixSort::SortPairs(tmp3, sort_tmp, (const unsigned*)cell, cell2, (const int*)tri, tri2, (int)H, 0,
                                  bits, st);
  cudaMemsetAsync(cnt, 0, (size_t)(H + 1) * 4, st);
  cub::DeviceRunLengthEncode::Encode(tmp3, rle_tmp, (const unsigned*)cell2, ucell, cnt, nrun, (int)H, st);
  if (read_back(fn, nrun, &U, 1, st)) return -1;
  // counts -> offsets[U + 1] (cnt[U] is 0)
  cub::DeviceScan::ExclusiveSum(tmp3, scan_tmp, cnt, cnt, (int)U + 1, st);
  // 4. out: cells uint32[U] | offsets int32[U + 1] | triangles int32[H]
  char* out = alloc(out_user, (size_t)(2 * U + 1 + H) * 4);
  if (!out) return fail(fn, "output allocation failed");
  cudaMemcpyAsync(out, ucell, (size_t)U * 4, cudaMemcpyDeviceToDevice, st);
  cudaMemcpyAsync(out + (size_t)U * 4, cnt, (size_t)(U + 1) * 4, cudaMemcpyDeviceToDevice, st);
  cudaMemcpyAsync(out + (size_t)(2 * U + 1) * 4, tri2, (size_t)H * 4, cudaMemcpyDeviceToDevice, st);
  return launched(fn) ? -1 : U;
}

int gsr_voxel_colors(int64_t ncell, const unsigned* cells, const int* offsets, const int* tris, int res,
                     double voxel_size, const double* verts, const int64_t* faces, const float* colors, float* rgb,
                     void* stream) {
  const char* fn = "gsr_voxel_colors";
  if (!count_ok(fn, ncell, "ncell")) return -1;
  if (res < 1 || res > 1024) return fail(fn, "res must be in 1..1024");
  if (!cells || !offsets || !tris || !verts || !faces || !colors || !rgb)
    return fail(fn, "cells, offsets, tris, verts, faces, colors and rgb are required");
  k_vox_colors<<<blocks(ncell, 128), 128, 0, (cudaStream_t)stream>>>(
      (int)ncell, cells, offsets, tris, res, voxel_size, verts, reinterpret_cast<const long long*>(faces), colors, rgb);
  return launched(fn);
}

}  // extern "C"
