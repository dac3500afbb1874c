// The photometric training loss of graphdeco's train.py, (1 - lambda) L1 + lambda (1 - SSIM) (DESIGN.md §7f): one
// forward kernel that gives, per CTA, the partial sums of |x - y| and of the SSIM map S (and, when a gradient is
// wanted, the three maps D0, D1, D2 the backward convolves), one reduction of those partials, and one backward kernel.
// The window is graphdeco's create_window(11, C): the float32 taps g of gaussian(11, 1.5) applied as g g^T in two 1D
// passes over a tile staged with a zero-filled 5-pixel halo, i.e. conv2d(padding=5) per (image, channel) plane.
//   mu1 = w*x   mu2 = w*y   s1 = w*(x x) - mu1^2   s2 = w*(y y) - mu2^2   s12 = w*(x y) - mu1 mu2
//   A1 = 2 mu1 mu2 + C1   A2 = 2 s12 + C2   B1 = mu1^2 + mu2^2 + C1   B2 = s1 + s2 + C2   S = A1 A2 / (B1 B2)
//   D0 = S (2 mu2 / A1 - 2 mu1 / B1 + 2 mu1 / B2 - 2 mu2 / A2)   D1 = -S / B2   D2 = 2 S / A2
//   dSum(S)/dx = w*D0 + 2 x (w*D1) + y (w*D2)        dSum|x - y|/dx = sign(x - y)
// The five window sums and everything up to the maps are formed in double: in float32, E[x x] - mu^2 of a flat region
// near 0.75 loses ~1e-7, which is 1e-4 of C2 and so of S.  The backward's window sums are float32 and its last line is
// double, where the products of two floats are exact (its terms are ~1/C2 and cancel to ~|x - y| / C2).  Every
// expression is the same on the x and the y side, so img1 == img2 gives mu1 = mu2, A1 = B1, A2 = B2, hence D0 = 0,
// w*D2 = -2 (w*D1) and a gradient of exactly zero.
#include "../../include/gsr.h"
#include "gsr_internal.cuh"

namespace gsr {

namespace {

constexpr int TX = 32, TY = 16;  // output pixels per CTA
constexpr int RAD = 5, TAPS = 2 * RAD + 1;
constexpr int SX = TX + 2 * RAD, SY = TY + 2 * RAD;  // staged tile with its halo
constexpr int THREADS = 256;                         // 32 x 8: each thread owns TY / 8 output rows of one column
constexpr int ROWS = TY / (THREADS / TX);
constexpr int WARPS = THREADS / 32;
constexpr int REDUCE_THREADS = 1024;
constexpr double C1 = 0.01 * 0.01, C2 = 0.03 * 0.03;  // graphdeco's Python floats

// graphdeco's gaussian(11, 1.5): exp(-(x - 5)^2 / 4.5) in float32, divided by its float32 sum
__device__ constexpr float kTap[TAPS] = {0x1.0d956cp-10f, 0x1.f1fe02p-8f, 0x1.26eb18p-5f, 0x1.bff0fep-4f,
                                         0x1.b43c3ep-3f,  0x1.106560p-2f, 0x1.b43c3ep-3f, 0x1.bff0fep-4f,
                                         0x1.26eb18p-5f,  0x1.f1fe02p-8f, 0x1.0d956cp-10f};

struct Tile {
  long long plane;  // (image, channel) plane of this CTA
  int x0, y0;       // its first output pixel
};

__device__ __forceinline__ Tile tile_of(int H, int W) {
  const int tx = (W + TX - 1) / TX, ty = (H + TY - 1) / TY;
  const long long per_plane = (long long)tx * ty;
  const long long b = blockIdx.x;
  const int t = (int)(b % per_plane);
  return {b / per_plane, (t % tx) * TX, (t / tx) * TY};
}

// NF planes of `src` (each `stride` floats apart) staged as [NF][SY][SX] with zeros outside the image
template <int NF>
__device__ __forceinline__ void stage(float (*s)[SY][SX], const float* src, long long stride, const Tile& t, int H,
                                      int W) {
  for (int i = threadIdx.x; i < SY * SX; i += THREADS) {
    const int r = i / SX, c = i - r * SX;
    const int gy = t.y0 - RAD + r, gx = t.x0 - RAD + c;
    const bool in = gy >= 0 && gy < H && gx >= 0 && gx < W;
    const long long o = (long long)gy * W + gx;
#pragma unroll
    for (int f = 0; f < NF; f++) s[f][r][c] = in ? src[f * stride + o] : 0.f;
  }
}

// window sum of output pixel (ry, c) over the horizontal sums h[.][SY][TX]
template <typename T>
__device__ __forceinline__ T vsum(const T (*h)[TX], int ry, int c) {
  T v = 0;
#pragma unroll
  for (int k = 0; k < TAPS; k++) v = fma((T)kTap[k], h[ry + k][c], v);
  return v;
}

// fixed-order CTA sum of one double per thread (result valid in thread 0)
__device__ __forceinline__ double cta_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) red[warp] = v;
  __syncthreads();
  v = 0.0;
  if (threadIdx.x == 0)
    for (int k = 0; k < (int)(blockDim.x >> 5); k++) v += red[k];
  __syncthreads();
  return v;
}

struct SsimFwdArgs {
  int H, W;
  long long plane_px;  // H * W
  long long maps_stride;  // planes * H * W: distance between D0, D1 and D2
  const float *x, *y;
  float* maps;         // [3][planes][H][W], or NULL
  double* cta_sums;    // [2][gridDim.x]: sum |x - y|, sum S of each CTA
};

__global__ void __launch_bounds__(THREADS) k_ssim_fwd(const SsimFwdArgs a) {
  __shared__ float s[2][SY][SX];
  __shared__ double h[5][SY][TX];  // horizontal window sums of x, y, x x, y y, x y
  __shared__ double red[WARPS];
  const Tile t = tile_of(a.H, a.W);
  const long long base = t.plane * a.plane_px;
  stage<1>(s, a.x + base, 0, t, a.H, a.W);
  stage<1>(s + 1, a.y + base, 0, t, a.H, a.W);
  __syncthreads();
  for (int i = threadIdx.x; i < SY * TX; i += THREADS) {
    const int r = i / TX, c = i - r * TX;
    double m1 = 0.0, m2 = 0.0, xx = 0.0, yy = 0.0, xy = 0.0;
#pragma unroll
    for (int k = 0; k < TAPS; k++) {
      const double x = s[0][r][c + k], y = s[1][r][c + k];
      m1 = fma((double)kTap[k], x, m1);
      m2 = fma((double)kTap[k], y, m2);
      xx = fma((double)kTap[k], x * x, xx);  // exact: a product of two floats
      yy = fma((double)kTap[k], y * y, yy);
      xy = fma((double)kTap[k], x * y, xy);
    }
    h[0][r][c] = m1; h[1][r][c] = m2; h[2][r][c] = xx; h[3][r][c] = yy; h[4][r][c] = xy;
  }
  __syncthreads();
  const int c = threadIdx.x % TX;
  double l1 = 0.0, ss = 0.0;
#pragma unroll
  for (int j = 0; j < ROWS; j++) {
    const int ry = threadIdx.x / TX + j * (THREADS / TX);
    const int gx = t.x0 + c, gy = t.y0 + ry;
    if (gx >= a.W || gy >= a.H) continue;
    const double mu1 = vsum(h[0], ry, c), mu2 = vsum(h[1], ry, c);
    const double exx = vsum(h[2], ry, c), eyy = vsum(h[3], ry, c), exy = vsum(h[4], ry, c);
    const double mu1sq = __dmul_rn(mu1, mu1), mu2sq = __dmul_rn(mu2, mu2), mu12 = __dmul_rn(mu1, mu2);
    const double s1 = __dsub_rn(exx, mu1sq), s2 = __dsub_rn(eyy, mu2sq), s12 = __dsub_rn(exy, mu12);
    const double A1 = __dadd_rn(2.0 * mu12, C1), A2 = __dadd_rn(2.0 * s12, C2);
    const double B1 = __dadd_rn(__dadd_rn(mu1sq, mu2sq), C1), B2 = __dadd_rn(__dadd_rn(s1, s2), C2);
    const double S = __ddiv_rn(__dmul_rn(A1, A2), __dmul_rn(B1, B2));
    const float x = s[0][ry + RAD][c + RAD], y = s[1][ry + RAD][c + RAD];
    l1 += (double)fabsf(__fsub_rn(x, y));
    ss += S;
    if (a.maps) {
      const double m2x = 2.0 * mu2, m1x = 2.0 * mu1;
      const double d = __dsub_rn(__dadd_rn(__dsub_rn(__ddiv_rn(m2x, A1), __ddiv_rn(m1x, B1)), __ddiv_rn(m1x, B2)),
                                 __ddiv_rn(m2x, A2));
      const long long o = base + (long long)gy * a.W + gx;
      a.maps[o] = (float)__dmul_rn(S, d);
      a.maps[a.maps_stride + o] = (float)-__ddiv_rn(S, B2);
      a.maps[2 * a.maps_stride + o] = (float)__ddiv_rn(2.0 * S, A2);
    }
  }
  l1 = cta_sum(l1, red);
  ss = cta_sum(ss, red);
  if (threadIdx.x == 0) {
    a.cta_sums[blockIdx.x] = l1;
    a.cta_sums[gridDim.x + blockIdx.x] = ss;
  }
}

// sums[0] = sum |x - y|, sums[1] = sum S over the n CTAs' sums, in one fixed order
__global__ void __launch_bounds__(REDUCE_THREADS) k_ssim_reduce(const double* __restrict__ cta_sums, int n,
                                                                float* __restrict__ sums) {
  __shared__ double red[REDUCE_THREADS / 32];
  double l1 = 0.0, ss = 0.0;
  for (int i = threadIdx.x; i < n; i += REDUCE_THREADS) {
    l1 += cta_sums[i];
    ss += cta_sums[n + i];
  }
  l1 = cta_sum(l1, red);
  ss = cta_sum(ss, red);
  if (threadIdx.x == 0) {
    sums[0] = (float)l1;
    sums[1] = (float)ss;
  }
}

struct SsimBwdArgs {
  int H, W;
  long long plane_px, maps_stride;
  const float *x, *y, *maps;
  const float* d_sums;  // dL/d sum|x - y|, dL/d sum S
  float* d_x;
};

__global__ void __launch_bounds__(THREADS) k_ssim_bwd(const SsimBwdArgs a) {
  __shared__ float s[3][SY][SX];
  __shared__ float h[3][SY][TX];
  const Tile t = tile_of(a.H, a.W);
  const long long base = t.plane * a.plane_px;
  stage<3>(s, a.maps + base, a.maps_stride, t, a.H, a.W);
  __syncthreads();
  for (int i = threadIdx.x; i < SY * TX; i += THREADS) {
    const int r = i / TX, c = i - r * TX;
    float v0 = 0.f, v1 = 0.f, v2 = 0.f;
#pragma unroll
    for (int k = 0; k < TAPS; k++) {
      v0 = fmaf(kTap[k], s[0][r][c + k], v0);
      v1 = fmaf(kTap[k], s[1][r][c + k], v1);
      v2 = fmaf(kTap[k], s[2][r][c + k], v2);
    }
    h[0][r][c] = v0; h[1][r][c] = v1; h[2][r][c] = v2;
  }
  __syncthreads();
  const float g_l1 = a.d_sums[0], g_s = a.d_sums[1];
  const int c = threadIdx.x % TX;
#pragma unroll
  for (int j = 0; j < ROWS; j++) {
    const int ry = threadIdx.x / TX + j * (THREADS / TX);
    const int gx = t.x0 + c, gy = t.y0 + ry;
    if (gx >= a.W || gy >= a.H) continue;
    const long long o = base + (long long)gy * a.W + gx;
    const float x = a.x[o], y = a.y[o];
    const float w0 = vsum(h[0], ry, c), w1 = vsum(h[1], ry, c), w2 = vsum(h[2], ry, c);
    const double gs = (double)w0 + 2.0 * (double)x * w1 + (double)y * w2;
    const float sgn = (float)((x > y) - (x < y));
    a.d_x[o] = (float)((double)g_l1 * sgn + (double)g_s * gs);
  }
}

// the checks every entry point makes before any work; -> number of CTAs, or -1 with the error text set
long long ssim_grid(const char* entry, long long planes, int H, int W) {
  if (planes < 1 || H < 1 || W < 1) return fail(entry, "planes, H and W must be >= 1");
  // 3 * planes * H * W: the elements of the D maps
  if (planes > INT64_MAX / 3 / H / W) return fail(entry, "element count overflows int64");
  const long long tiles = (long long)((W + TX - 1) / TX) * ((H + TY - 1) / TY);
  if (planes > 0x7fffffffll / tiles) return fail(entry, "too many tiles for one grid (planes x tiles must fit in int32)");
  return planes * tiles;
}

}  // namespace

}  // namespace gsr

using namespace gsr;

extern "C" {

size_t gsr_ssim_scratch_bytes(int64_t planes, int H, int W) {
  const long long n = ssim_grid("gsr_ssim_scratch_bytes", planes, H, W);
  return n < 0 ? 0 : (size_t)n * 2 * sizeof(double);
}

int gsr_ssim_forward(int64_t planes, int H, int W, const float* img1, const float* img2, float* partials,
                     void* scratch, float* sums, void* stream) {
  const long long n = ssim_grid("gsr_ssim_forward", planes, H, W);
  if (n < 0) return -1;
  if (!img1 || !img2 || !scratch || !sums) return fail("gsr_ssim_forward", "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  SsimFwdArgs a{};
  a.H = H; a.W = W; a.plane_px = (long long)H * W; a.maps_stride = planes * a.plane_px;
  a.x = img1; a.y = img2; a.maps = partials; a.cta_sums = (double*)scratch;
  k_ssim_fwd<<<(unsigned)n, THREADS, 0, st>>>(a);
  k_ssim_reduce<<<1, REDUCE_THREADS, 0, st>>>(a.cta_sums, (int)n, sums);
  return launched("gsr_ssim_forward");
}

int gsr_ssim_backward(int64_t planes, int H, int W, const float* img1, const float* img2, const float* partials,
                      const float* d_sums, float* d_img1, void* stream) {
  const long long n = ssim_grid("gsr_ssim_backward", planes, H, W);
  if (n < 0) return -1;
  if (!img1 || !img2 || !partials || !d_sums || !d_img1) return fail("gsr_ssim_backward", "null pointer");
  SsimBwdArgs a{};
  a.H = H; a.W = W; a.plane_px = (long long)H * W; a.maps_stride = planes * a.plane_px;
  a.x = img1; a.y = img2; a.maps = partials; a.d_sums = d_sums; a.d_x = d_img1;
  k_ssim_bwd<<<(unsigned)n, THREADS, 0, (cudaStream_t)stream>>>(a);
  return launched("gsr_ssim_backward");
}

}  // extern "C"
