// Per-tile alpha compositing, forward and backward: replaces renderCUDA
// ($RAST/cuda_rasterizer/forward.cu:261-397 and backward.cu:415-610).
//
// What is kept exactly (observable behaviour, SURVEY.md §8b): a pixel evaluates the Gaussians of its 16x16
// tile's sorted list in order, with the reference's per-pair arithmetic (same FMA contraction as its SASS,
// precise expf), thresholds (power>0, alpha<1/255, T<1e-4, median at T crossing 0.5), contributor counting
// and un-normalised depth / no-background colour outputs.
//
// What is different (H100):
//  * a dedicated producer warp walks the tile's sorted index list and stages the 48-byte splat records of
//    the next batches into a shared-memory ring with asynchronous 16-byte copies (cp.async, completion on an
//    mbarrier), NSTAGE batches ahead of the consumer warps -- no CTA-wide barrier in the loop, and
//    rgb/depth come from shared memory instead of per-pair global loads (forward.cu:365-366).  Only the
//    part of the list a tile really consumes is ever gathered (early termination / n_contrib bound).  All
//    waits are blocking mbarrier waits (no polling of shared flags): when every pixel of a tile is finished
//    the producer completes the next, never-gathered batch with plain arrivals (a "poison" batch) and the
//    parked consumer warps leave through it;
//  * every 8x4 pixel block first tests the staged Gaussians against its rectangle with a conservative bound
//    on alpha (minimum of the conic form over the rectangle, threshold 2 ln(255 o) precomputed per Gaussian);
//    only survivors are evaluated.  A pair is skipped only if the reference would `continue` past it for
//    every pixel of the block (alpha < 1/255), so results are unchanged while most evaluations disappear;
//  * backward: one lane owns NSUB pixels (one in each of the warp's NSUB 8x4 blocks) and sums a Gaussian's
//    gradient contributions over its own pixels in registers before the warp-level reduction, so the
//    transposed shuffle butterfly + predicated red.global run once per (warp region, Gaussian) instead of
//    once per (8x4 block, Gaussian) -- and instead of 11-12 atomicAdd per (pixel, Gaussian) pair
//    (backward.cu:559-607).  The per-pair arithmetic is re-derived for instruction count (see the kernel body):
//    one scalar "behind" recurrence for all five blended channels, and the mean / conic gradients are
//    accumulated as raw moments of u = dL/dG * G (sum u dx, u dy, u dx^2, u dx dy, u dy^2) that the
//    per-Gaussian kernel turns into dL/dmean2D and dL/dconic.  Traversal starts at the tile's largest
//    n_contrib instead of the end of the list.
#include "../../include/gsr.h"
#include "gsr_internal.cuh"
#include <cstdlib>
#include <cstring>

namespace gsr {

namespace {

// GSR_RB / GSR_NSTAGE: overridden only by the stress build of tests/test_gpu_ring_stress.py (1 stage of 32 records: every
// batch is a wrap-around of the ring, so a protocol slip shows up as wrong pixels instead of hiding behind slack)
#ifndef GSR_RB
#define GSR_RB 128
#endif
#ifndef GSR_NSTAGE
#define GSR_NSTAGE 4
#endif
constexpr int RB = GSR_RB;                    // records per pipeline stage (a multiple of 32)
constexpr int NSTAGE = GSR_NSTAGE;            // ring depth: consumer warps may drift this many batches apart
static_assert(RB % 32 == 0 && RB >= 32 && NSTAGE >= 1, "ring geometry");
constexpr int STAGE_F4 = RB * SPLAT_F4;       // float4 per stage (6 KB)
constexpr int NBLK = TILE_PIX / 32;           // 8 blocks of 8x4 pixels per tile
constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// asynchronous 16-byte global->shared copy (LDGSTS, L2 only) and its completion hook on an mbarrier
__device__ __forceinline__ void cp_async16(void* dst_smem, const void* src_gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst_smem)), "l"(src_gmem) : "memory");
}
__device__ __forceinline__ void cp_async_arrive(unsigned long long* bar) {
  // the arrival fires once all of this thread's earlier cp.async have landed; .noinc: counted in the init value
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// producer warp: gather `cnt` records listed in ids[0,cnt) into a stage
__device__ __forceinline__ void stage_gather(float4* dst, const float4* __restrict__ splat,
                                             const uint32_t* __restrict__ ids, int cnt, int lane,
                                             unsigned long long* full) {
  for (int r = lane; r < cnt; r += 32) {
    const float4* src = splat + (size_t)ids[r] * SPLAT_F4;
    cp_async16(dst + r * SPLAT_F4 + 0, src + 0);
    cp_async16(dst + r * SPLAT_F4 + 1, src + 1);
    cp_async16(dst + r * SPLAT_F4 + 2, src + 2);
  }
  cp_async_arrive(full);
}
// ---- TMA bulk-copy staging (opt-in, GSR_FWD_TMA=1; DESIGN.md 3.2) ---------------------------------------------
// One cp.async.bulk per record: the TMA engine copies the 48 contiguous bytes of splat[id] into the stage (both ends
// 16-byte aligned), and the copy completes its bytes on the stage's `full` barrier.  Same stage layout as the
// LDGSTS flavour.
__device__ __forceinline__ void tma_copy(void* dst_smem, const void* src_gmem, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// producer warp, TMA flavour: lane l copies records l, l+32, ...; each lane first announces its bytes with its one
// arrival on `full` (initialised for 32), so the phase completes once all 32 lanes arrived and every byte landed
__device__ __forceinline__ void stage_gather_tma(float4* dst, const float4* __restrict__ splat,
                                                 const uint32_t* __restrict__ ids, int cnt, int lane,
                                                 unsigned long long* full) {
  const int mine = cnt > lane ? (cnt - lane + 31) / 32 : 0;
  mbar_arrive_expect(full, (unsigned)(mine * SPLAT_BYTES));
  for (int r = lane; r < cnt; r += 32) tma_copy(dst + r * SPLAT_F4, splat + (size_t)ids[r] * SPLAT_F4, SPLAT_BYTES, full);
}

// forward.cu:343-356 with the contraction of the reference SASS (SURVEY.md A.4): the Gaussian's exponent and alpha at
// one pixel.  Shared by the forward and the contribution pass, so both take the same blend decisions bit for bit.
__device__ __forceinline__ float pair_power(const float4 q0, const float4 q1, float pxf, float pyf) {
  const float dx = q0.x - pxf, dy = q0.y - pyf;
  const float t1 = __fmul_rn(__fmul_rn(dy, q1.x), dy);
  const float t2 = __fmul_rn(dx, q0.z);
  const float t3 = __fmul_rn(__fmul_rn(dx, q0.w), dy);
  return __fmaf_rn(__fmaf_rn(dx, t2, t1), -0.5f, -t3);
}
__device__ __forceinline__ float pair_alpha(const float4 q1, float power) {
  return fminf(0.99f, __fmul_rn(q1.y, expf(power)));
}

__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try(unsigned long long* bar, unsigned parity) {
  unsigned ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// RELAXED: the waiter has nothing urgent to do (a warp whose pixels are all finished only keeps releasing stages):
// back off with nanosleep between polls so it does not take issue slots from the warps that still composite.
template <bool RELAXED = false>
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
  if (RELAXED) {
    while (!mbar_try(bar, parity)) __nanosleep(400);
    return;
  }
  const unsigned b = smem_u32(bar);
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\n"
      "bra WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(b),
      "r"(parity)
      : "memory");
}

// ---------------------------------------------------------------------------------------------
// Shared-memory ring shared by both kernels: NSTAGE record batches, `full` barriers completed by the
// producer lanes' cp.async arrivals, `empty` barriers by one arrival per consumer warp.  The last warp of the
// CTA is the producer: it refills a stage as soon as every consumer warp released it.
// Consumer warps never meet at a CTA-wide barrier inside the loop, so a block with little work does not
// wait for a crowded one batch by batch.
// ---------------------------------------------------------------------------------------------
template <int STAGE>
struct RingT {
  float4 buf[NSTAGE][STAGE];
  unsigned long long full[NSTAGE];
  unsigned long long empty[NSTAGE];
  unsigned ndone;           // forward: consumer warps that have no live pixel left
  int stop_at;              // forward: index of the poison batch (the producer stopped before gathering it)
  unsigned maxc[NBLK];
};

typedef RingT<STAGE_F4> Ring;

template <int STAGE>
__device__ __forceinline__ void ring_init(RingT<STAGE>& r, int consumers) {
  if (threadIdx.x == 0) {
#pragma unroll
    for (int s = 0; s < NSTAGE; s++) { mbar_init(&r.full[s], 32); mbar_init(&r.empty[s], consumers); }
    r.ndone = 0;
    r.stop_at = -1;
    fence_mbar_init();
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------
// forward: 8 consumer warps (one 8x4 block each) + 1 producer warp
// ---------------------------------------------------------------------------------------------
constexpr int FWD_THREADS = TILE_PIX + 32;

template <bool TMA>
__global__ void __launch_bounds__(FWD_THREADS) k_render_fwd(int W, int H, int gx, ImageView im, BinView bin,
                                                            const float4* __restrict__ splat,
                                                            float* __restrict__ out_color,
                                                            float* __restrict__ out_depth,
                                                            float* __restrict__ out_median,
                                                            float* __restrict__ out_opacity) {
  __shared__ __align__(128) Ring ring;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int tile = (int)im.tile_order[blockIdx.x], tx = tile % gx, ty = tile / gx;  // longest tiles first
  const uint2 range = im.tile_range[tile];
  const int n = (int)(range.y - range.x);
  const int nb = (n + RB - 1) / RB;
  const uint32_t* ids = bin.point_list + range.x;
  ring_init(ring, NBLK);

  if (warp == NBLK) {
    // ---------------- producer warp ----------------
    int issued = 0;
    for (int b = 0; b < nb; b++) {
      const int s = b % NSTAGE;
      int stop = 0;
      if (lane == 0) {
        // the ring is NSTAGE batches deep: the refill can afford the back-off of a relaxed wait
        if (b >= NSTAGE) mbar_wait<true>(&ring.empty[s], (unsigned)((b / NSTAGE - 1) & 1));
        stop = *(volatile unsigned*)&ring.ndone == NBLK;  // every pixel of the tile is finished
      }
      if (__shfl_sync(FULL, stop, 0)) break;
      if (TMA) stage_gather_tma(ring.buf[s], splat, ids + b * RB, min(RB, n - b * RB), lane, &ring.full[s]);
      else stage_gather(ring.buf[s], splat, ids + b * RB, min(RB, n - b * RB), lane, &ring.full[s]);
      issued = b + 1;
    }
    // every copy must have landed before the CTA's shared memory is released
    for (int b = max(0, issued - NSTAGE); b < issued; b++) mbar_wait(&ring.full[b % NSTAGE], (unsigned)((b / NSTAGE) & 1));
    if (issued < nb) {
      // poison batch: consumers parked on the batch that will never be gathered leave through it
      if (lane == 0) *(volatile int*)&ring.stop_at = issued;
      __syncwarp();
      mbar_arrive(&ring.full[issued % NSTAGE]);  // 32 plain arrivals complete the phase
    }
    return;
  }

  // ---------------- consumers: warp w owns the 8x4 block at (w&1, w>>1) ----------------
  const int sx0 = tx * TILE_X + (warp & 1) * 8, sy0 = ty * TILE_Y + (warp >> 1) * 4;
  const int px = sx0 + (lane & 7), py = sy0 + (lane >> 3);
  const bool inside = px < W && py < H;
  const float pxf = (float)px, pyf = (float)py;
  const float rx0 = (float)sx0, ry0 = (float)sy0;
  const float rx1 = (float)min(sx0 + 7, W - 1), ry1 = (float)min(sy0 + 3, H - 1);

  // A finished pixel (T would drop below 1e-4, forward.cu:357-362, or outside the image) is marked by the SIGN of T:
  // T * (1 - alpha) stays negative, so it keeps failing the same test and never blends again.
  float T = inside ? 1.0f : -1.0f, C0 = 0.f, C1 = 0.f, C2 = 0.f, D = 0.f;
  float med_d = 15.0f, med_w = 0.f, med_id = 0.f;  // forward.cu:310-312
  unsigned last_contributor = 0;
  bool warp_done = __all_sync(FULL, T < 0.f);
  if (warp_done && lane == 0) atomicAdd(&ring.ndone, 1u);

  for (int b = 0; b < nb; b++) {
    const int s = b % NSTAGE;
    if (warp_done) {
      // nothing left for this warp: keep releasing stages (without competing for issue slots) until the producer stops
      mbar_wait<true>(&ring.full[s], (unsigned)((b / NSTAGE) & 1));
      if (*(volatile int*)&ring.stop_at == b) break;
      if (lane == 0) mbar_arrive(&ring.empty[s]);
      continue;
    }
    mbar_wait(&ring.full[s], (unsigned)((b / NSTAGE) & 1));
    const int cnt = min(RB, n - b * RB);
    const float4* sb = ring.buf[s];
    for (int base = 0; base < cnt; base += 32) {
      const int j = base + lane;
      bool keep = false;
      if (j < cnt) {
        const float4* cr = sb + j * SPLAT_F4;
        keep = may_touch(cull_prep(cr[0], cr[1], cr[2].w), rx0, ry0, rx1, ry1);
      }
      unsigned mask = __ballot_sync(FULL, keep);
      const unsigned pos0 = (unsigned)(b * RB + base + 1);
      while (mask) {
        const int bit = __ffs(mask) - 1;
        mask &= mask - 1;
        const float4* rec = sb + (base + bit) * SPLAT_F4;
        const float4 q0 = rec[0], q1 = rec[1];
        const float power = pair_power(q0, q1, pxf, pyf);
        if (power > 0.0f) continue;
        const float alpha = pair_alpha(q1, power);
        if (alpha < 1.0f / 255.0f) continue;
        const float test_T = __fmul_rn(T, __fsub_rn(1.0f, alpha));
        if (test_T < 0.0001f) { T = -fabsf(T); continue; }
        const float4 q2 = rec[2];
        C0 = __fmaf_rn(T, __fmul_rn(alpha, q1.w), C0);
        C1 = __fmaf_rn(T, __fmul_rn(alpha, q2.x), C1);
        C2 = __fmaf_rn(T, __fmul_rn(alpha, q2.y), C2);
        D = __fmaf_rn(T, __fmul_rn(alpha, q1.z), D);
        if (T > 0.5f && test_T < 0.5f) {
          med_d = q1.z;
          med_w = __fmul_rn(alpha, T);
          med_id = (float)__float_as_int(q2.z);
        }
        T = test_T;
        last_contributor = pos0 + (unsigned)bit;
      }
      warp_done = __all_sync(FULL, T < 0.f);
      if (warp_done) break;
    }
    __syncwarp();
    if (lane == 0) {
      if (warp_done) atomicAdd(&ring.ndone, 1u);
      mbar_arrive(&ring.empty[s]);
    }
  }

  if (inside) {
    const size_t pid = (size_t)py * W + px, HW = (size_t)W * H;
    const float Tf = fabsf(T);
    im.final_T[pid] = Tf;
    im.n_contrib[pid] = last_contributor;
    out_color[pid] = C0;  // no background blend (forward.cu:389-390)
    out_color[HW + pid] = C1;
    out_color[2 * HW + pid] = C2;
    out_depth[pid] = D;
    out_median[pid] = med_d;
    out_median[HW + pid] = med_w;
    out_median[2 * HW + pid] = med_id;
    out_opacity[pid] = 1 - Tf;
  }
  // largest n_contrib of the tile bounds the backward traversal
  const unsigned wmax = __reduce_max_sync(FULL, last_contributor);
  if (lane == 0) ring.maxc[warp] = wmax;
  asm volatile("bar.sync 1, %0;" ::"n"(TILE_PIX) : "memory");  // consumer warps only (the producer has left)
  if (tid == 0) {
    unsigned m = 0;
#pragma unroll
    for (int w = 0; w < NBLK; w++) m = max(m, ring.maxc[w]);
    im.tile_maxc[tile] = m;
  }
}

// ---------------------------------------------------------------------------------------------
// backward: 8 / NSUB consumer warps, each owning NSUB 8x4 blocks (lane = one pixel in every block), + producer
// ---------------------------------------------------------------------------------------------
// block s of warp w sits at (kx, ky) in units of (8, 4) pixels; regions are as square as possible:
//   NSUB 1: 8x4    NSUB 2: 8x8    (4: 16x8 and 8: the whole tile were measured too and are not instantiated)
template <int NSUB> __device__ __forceinline__ int blk_kx(int w, int s) { return NSUB <= 2 ? (w & 1) : (s & 1); }
template <int NSUB> __device__ __forceinline__ int blk_ky(int w, int s) {
  return NSUB == 1 ? (w >> 1) : NSUB == 2 ? (w >> 1) * 2 + s : NSUB == 4 ? w * 2 + (s >> 1) : (s >> 1);
}

#ifndef GSR_BWD_BOUND_EXTRA
#define GSR_BWD_BOUND_EXTRA 0
#endif
// 1 (default): the compositing backward evaluates exp with one ex2.approx; 0: precise expf (chosen by A/B)
#ifndef GSR_BWD_FASTEXP
#define GSR_BWD_FASTEXP 1
#endif
template <int NSUB, int MINB>
__global__ void __launch_bounds__((NBLK / NSUB) * 32 + 32 + (NSUB == 1 ? GSR_BWD_BOUND_EXTRA : 0), MINB)
k_render_bwd(int W, int H, int gx, const float* __restrict__ bg, ImageView im, BinView bin,
             const float4* __restrict__ splat, float* __restrict__ grad, const float* __restrict__ dL_dpix,
             const float* __restrict__ dL_ddepthpix, const float* __restrict__ dL_dmedpix,
             const float* __restrict__ dL_dopacpix) {
  constexpr int NCONS = NBLK / NSUB;
  __shared__ __align__(128) Ring ring;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int tile = (int)im.tile_order[blockIdx.x], tx = tile % gx, ty = tile / gx;  // longest tiles first
  const uint2 range = im.tile_range[tile];
  const int nmax = (int)min(im.tile_maxc[tile], range.y - range.x);
  if (nmax == 0) return;
  const int nb = (nmax + RB - 1) / RB;
  const uint32_t* ids = bin.point_list + range.x;
  ring_init(ring, NCONS);

  // batch b (counted from the back) covers list positions [lo_b, hi_b), hi_b = nmax - b*RB
  if (warp == NCONS) {
    for (int b = 0; b < nb; b++) {
      const int s = b % NSTAGE;
      if (b >= NSTAGE) {
        if (lane == 0) mbar_wait<true>(&ring.empty[s], (unsigned)((b / NSTAGE - 1) & 1));
        __syncwarp();
      }
      const int hi = nmax - b * RB, lo = max(0, hi - RB);
      stage_gather(ring.buf[s], splat, ids + lo, hi - lo, lane, &ring.full[s]);
    }
    // the consumers wait on every batch, so all copies have landed when they leave; nothing to drain
    return;
  }

  // per-pixel state of the lane's NSUB pixels
  const size_t HW = (size_t)W * H;
  const int lx = lane & 7, ly = lane >> 3;
  const int bx0 = tx * TILE_X, by0 = ty * TILE_Y;
  float T[NSUB], Q[NSUB], g0[NSUB], g1[NSUB], g2[NSUB], gD[NSUB], gO[NSUB], gM[NSUB];
  int lastc[NSUB], maxs[NSUB];
  int warp_max = 0;
#pragma unroll
  for (int s = 0; s < NSUB; s++) {
    const int px = bx0 + blk_kx<NSUB>(warp, s) * 8 + lx, py = by0 + blk_ky<NSUB>(warp, s) * 4 + ly;
    const bool inside = px < W && py < H;
    const size_t pid = (size_t)py * W + px;
    T[s] = inside ? im.final_T[pid] : 0.f;
    lastc[s] = inside ? (int)im.n_contrib[pid] : 0;
    g0[s] = g1[s] = g2[s] = gD[s] = gO[s] = gM[s] = 0.f;
    if (inside) {
      g0[s] = dL_dpix[pid]; g1[s] = dL_dpix[HW + pid]; g2[s] = dL_dpix[2 * HW + pid];
      gD[s] = dL_ddepthpix[pid];
      gO[s] = dL_dopacpix[pid];
      gM[s] = dL_dmedpix[pid];  // channel 0 of the median-depth gradient (quirk 4)
    }
    // Q = (sum of s_i w_i over the contributors behind the current one) + T_final * (bg . dL_dpix): the second
    // term is the background contribution of backward.cu:584-587, folded into the same recurrence
    float bg_dot = 0.f;
    bg_dot += bg[0] * g0[s]; bg_dot += bg[1] * g1[s]; bg_dot += bg[2] * g2[s];
    Q[s] = T[s] * bg_dot;
    maxs[s] = (int)__reduce_max_sync(FULL, (unsigned)lastc[s]);
    warp_max = max(warp_max, maxs[s]);
  }
  // which lane publishes which reduced component (see the butterfly below): even lanes; of those with bit 1 set (they
  // all hold component 4 / 9) only lanes 2 and 18
  const bool pub = (lane & 1) == 0 && ((lane & 2) == 0 || (lane & 12) == 0);
  const int slot = ((lane & 16) ? 5 : 0) + ((lane & 2) ? 4 : ((lane & 4) ? 2 : 0) + ((lane & 8) ? 1 : 0));
  // kept opaque so that the compiler holds them in registers instead of rebuilding them from %tid for every pair
  unsigned lanebits = (unsigned)lane | (pub ? 32u : 0u);
  float* gslot = grad + slot;
  asm volatile("" : "+r"(lanebits), "+l"(gslot));

  for (int b = 0; b < nb; b++) {
    const int st = b % NSTAGE;
    mbar_wait(&ring.full[st], (unsigned)((b / NSTAGE) & 1));
    const int hi = nmax - b * RB, lo = max(0, hi - RB), cnt = hi - lo;
    const float4* sb = ring.buf[st];
    if (lo < warp_max) {
      for (int base = 0; base < cnt; base += 32) {
        const int j = cnt - 1 - (base + lane);  // lane 0 = farthest entry of this chunk
        unsigned m[NSUB];
        {
          CullRec cr;
          cr.live = false;
          if (j >= 0 && lo + j < warp_max) cr = cull_prep(sb[j * SPLAT_F4], sb[j * SPLAT_F4 + 1], sb[j * SPLAT_F4 + 2].w);
#pragma unroll
          for (int s = 0; s < NSUB; s++) {
            const int rxi = bx0 + blk_kx<NSUB>(warp, s) * 8, ryi = by0 + blk_ky<NSUB>(warp, s) * 4;
            bool keep = false;
            if (cr.live && lo + j < maxs[s] && rxi < W && ryi < H)
              keep = may_touch(cr, (float)rxi, (float)ryi, (float)min(rxi + 7, W - 1), (float)min(ryi + 3, H - 1));
            m[s] = __ballot_sync(FULL, keep);
          }
        }
        unsigned any = m[0];
#pragma unroll
        for (int s = 1; s < NSUB; s++) any |= m[s];
        while (any) {
          const int bit = __ffs(any) - 1;
          any &= any - 1;
          const int jj = cnt - 1 - (base + bit);
          const int pos = lo + jj;
          const float4* rec = sb + jj * SPLAT_F4;
          const float4 q0 = rec[0], q1 = rec[1], q2 = rec[2];
          // v0-2 colour, v3 depth, v4 opacity, v5-6 sum u dx / u dy, v7-9 sum u dx^2 / u dx dy / u dy^2
          // (one pixel per lane: every component is assigned before it is read, see `acc` below)
          float v0, v1, v2, v3, v4, v5, v6, v7, v8, v9;
          if (NSUB > 1) v0 = v1 = v2 = v3 = v4 = v5 = v6 = v7 = v8 = v9 = 0.f;
          bool contrib = false;
#pragma unroll
          for (int s = 0; s < NSUB; s++) {
            if (NSUB > 1 && !((m[s] >> bit) & 1u)) continue;  // warp-uniform
            const float dx = q0.x - (float)(bx0 + blk_kx<NSUB>(warp, s) * 8 + lx);
            const float dy = q0.y - (float)(by0 + blk_ky<NSUB>(warp, s) * 4 + ly);
            const float t1 = __fmul_rn(__fmul_rn(dy, q1.x), dy);
            const float t2 = __fmul_rn(dx, q0.z);
            const float t3 = __fmul_rn(__fmul_rn(dx, q0.w), dy);
            const float power = __fmaf_rn(__fmaf_rn(dx, t2, t1), -0.5f, -t3);
            // branch-free form: a lane whose pixel does not take this Gaussian (backward.cu:520-537: at or beyond
            // n_contrib, power > 0, alpha < 1/255) runs the same arithmetic with G = 0, which makes its alpha, weight
            // and every accumulated term exactly zero and leaves its T and Q untouched (1 / (1 - 0) == 1 exactly)
            // one pixel per lane: the sums start here, so plain products (no zero-initialised accumulators)
            auto acc = [](float x, float y, float z) { return NSUB == 1 ? x * y : fmaf(x, y, z); };
#if GSR_BWD_FASTEXP
            // exp as ONE ex2.approx of power * log2(e) (2 instructions instead of expf's 10; relative error ~4e-7 for
            // the powers that pass the alpha test: gradient tolerance is 1e-3).  A pair whose alpha sits within that
            // error of 1/255 may be taken here and skipped by the forward (or the reverse): one 0.4 % step of one
            // pixel's transmittance
            float G0;
            asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(G0) : "f"(power * 1.4426950408889634f));
#else
            const float G0 = expf(power);
#endif
            const float al0 = fminf(0.99f, q1.y * G0);
            const bool valid = (pos < lastc[s]) && !(power > 0.0f) && !(al0 < 1.0f / 255.0f);
            if (!__any_sync(FULL, valid)) continue;
            contrib = true;
            const float G = valid ? G0 : 0.f;
            const float alpha = valid ? al0 : 0.f;
            float inv;
            asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(inv) : "f"(1.f - alpha));
            const float Tb = T[s] * inv;
            const float w = alpha * Tb;
            const float sj = fmaf(q1.w, g0[s], fmaf(q2.x, g1[s], fmaf(q2.y, g2[s], fmaf(q1.z, gD[s], gO[s]))));
            const float dL_dalpha = fmaf(sj, Tb, -(Q[s] * inv));
            Q[s] = fmaf(sj, w, Q[s]);
            v0 = acc(w, g0[s], v0);
            v1 = acc(w, g1[s], v1);
            v2 = acc(w, g2[s], v2);
            v3 = acc(w, gD[s], v3);
            // backward.cu:566-569: the Gaussian at which T crosses 0.5 also receives the median-depth gradient
            // (never true for a masked lane: Tb == T there)
            if (Tb > 0.5f && T[s] < 0.5f) v3 += gM[s];
            v4 = acc(w, gO[s], v4);
            v4 = fmaf(G, dL_dalpha, v4);
            const float u = (q1.y * dL_dalpha) * G;
            const float ux = u * dx, uy = u * dy;
            v5 = NSUB == 1 ? ux : v5 + ux;
            v6 = NSUB == 1 ? uy : v6 + uy;
            v7 = acc(ux, dx, v7);
            v8 = acc(ux, dy, v8);
            v9 = acc(uy, dy, v9);
            T[s] = Tb;
          }
          if (!contrib) continue;
          // transposed butterfly over all ten components: every stage halves what a lane still carries (two of its
          // values form one, the partner lane keeps the other half), an odd one out is reduced in place --
          // 5 + 3 + 2 + 1 + 1 = 12 shuffles -- and one lane per component ends up with its total in ONE register:
          //   bit 16 of the lane picks v0-4 / v5-9, then bit 1 = 0: component 2*bit2 + bit3, bit 1 = 1: component 4
          const bool h16 = lanebits & 16, h8 = lanebits & 8, h4 = lanebits & 4, h2 = lanebits & 2;
          float x0 = h16 ? v5 : v0, x1 = h16 ? v6 : v1, x2 = h16 ? v7 : v2, x3 = h16 ? v8 : v3, x4 = h16 ? v9 : v4;
          x0 += __shfl_xor_sync(FULL, h16 ? v0 : v5, 16);
          x1 += __shfl_xor_sync(FULL, h16 ? v1 : v6, 16);
          x2 += __shfl_xor_sync(FULL, h16 ? v2 : v7, 16);
          x3 += __shfl_xor_sync(FULL, h16 ? v3 : v8, 16);
          x4 += __shfl_xor_sync(FULL, h16 ? v4 : v9, 16);
          float y0 = h8 ? x1 : x0, y1 = h8 ? x3 : x2;
          y0 += __shfl_xor_sync(FULL, h8 ? x0 : x1, 8);
          y1 += __shfl_xor_sync(FULL, h8 ? x2 : x3, 8);
          x4 += __shfl_xor_sync(FULL, x4, 8);
          float z0 = h4 ? y1 : y0;
          z0 += __shfl_xor_sync(FULL, h4 ? y0 : y1, 4);
          x4 += __shfl_xor_sync(FULL, x4, 4);
          float r = h2 ? x4 : z0;
          r += __shfl_xor_sync(FULL, h2 ? z0 : x4, 2);
          r += __shfl_xor_sync(FULL, r, 1);
          // (red.global spelled out: behind the opaque pointer atomicAdd would take the generic-address path)
          if (lanebits & 32)
            asm volatile("red.global.add.f32 [%0], %1;" ::"l"(gslot + (size_t)__float_as_int(q2.z) * GRAD_F), "f"(r) : "memory");
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&ring.empty[st]);
  }
}

// ---------------------------------------------------------------------------------------------
// contribution statistics (gsr_contribution, DESIGN.md §7l): the forward's per-pixel walk replayed on its own buffers
// ---------------------------------------------------------------------------------------------
// A pixel whose walk ended on T (1 - alpha) < 1e-4 had T < CONTRIB_END_T when it ended: alpha <= 0.99 leaves
// 1 - alpha >= 0.0099999, so the product of a T >= 0.0101 stays above 1e-4 after rounding.  A pixel whose final T is at
// least this therefore never ended, and nothing behind its last contributor reached the transmittance test.
constexpr float CONTRIB_END_T = 0.0101f;
constexpr int CONTRIB_THREADS = TILE_PIX;  // one pixel per thread; warp w owns the forward's 8x4 block w
// weight fixed point: a blend weight w <= 0.99 becomes round(w 2^32) < 2^32, a per-view sum of at most 2^26 pixels
// stays below 2^58
constexpr float CONTRIB_FIX = 4294967296.0f;

__global__ void __launch_bounds__(CONTRIB_THREADS) k_render_contrib(int W, int H, int gx, ImageView im, BinView bin,
                                                                    const float4* __restrict__ splat,
                                                                    unsigned long long* __restrict__ fixed_w,
                                                                    unsigned long long* __restrict__ count,
                                                                    unsigned* __restrict__ max_w) {
  __shared__ float4 recs[CONTRIB_THREADS * SPLAT_F4];
  __shared__ unsigned cta_lim;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int tile = (int)im.tile_order[blockIdx.x], tx = tile % gx, ty = tile / gx;
  const uint2 range = im.tile_range[tile];
  const int n = (int)(range.y - range.x);
  if (n == 0) return;
  const uint32_t* ids = bin.point_list + range.x;

  const int sx0 = tx * TILE_X + (warp & 1) * 8, sy0 = ty * TILE_Y + (warp >> 1) * 4;
  const int px = sx0 + (lane & 7), py = sy0 + (lane >> 3);
  const bool inside = px < W && py < H;
  const float pxf = (float)px, pyf = (float)py;
  const float rx0 = (float)sx0, ry0 = (float)sy0;
  const float rx1 = (float)min(sx0 + 7, W - 1), ry1 = (float)min(sy0 + 3, H - 1);
  // list positions this pixel's walk can reach a transmittance test at: all of them if it may have ended, else up to
  // its last contributor (n_contrib is 1 + that position)
  int lim = 0;
  if (inside) {
    const size_t pid = (size_t)py * W + px;
    lim = im.final_T[pid] < CONTRIB_END_T ? n : min(n, (int)im.n_contrib[pid]);
  }
  const int warp_lim = (int)__reduce_max_sync(FULL, (unsigned)lim);
  if (tid == 0) cta_lim = 0;
  __syncthreads();
  if (lane == 0) atomicMax(&cta_lim, (unsigned)warp_lim);
  __syncthreads();
  const int nlim = (int)cta_lim;

  // the forward's state of this pixel: a finished pixel has T < 0 (never again reaches the test)
  float T = lim > 0 ? 1.0f : -1.0f;
  for (int b0 = 0; b0 < nlim; b0 += CONTRIB_THREADS) {
    const int cnt = min(CONTRIB_THREADS, nlim - b0);
    if (tid < cnt) {
      const float4* src = splat + (size_t)ids[b0 + tid] * SPLAT_F4;
      recs[tid * SPLAT_F4 + 0] = src[0];
      recs[tid * SPLAT_F4 + 1] = src[1];
      recs[tid * SPLAT_F4 + 2] = src[2];
    }
    __syncthreads();
    if (__any_sync(FULL, T > 0.f)) {
      for (int base = 0; base < cnt && b0 + base < warp_lim; base += 32) {
        const int j = base + lane;
        bool keep = false;
        if (j < cnt) {
          const float4* cr = recs + j * SPLAT_F4;
          keep = may_touch(cull_prep(cr[0], cr[1], cr[2].w), rx0, ry0, rx1, ry1);
        }
        unsigned mask = __ballot_sync(FULL, keep);
        while (mask) {
          const int bit = __ffs(mask) - 1;
          mask &= mask - 1;
          const float4* rec = recs + (base + bit) * SPLAT_F4;
          const float4 q0 = rec[0], q1 = rec[1];
          // the forward's decisions in its order: power > 0 and alpha < 1/255 skip the pair, then the pixel ends
          // (counted, no weight) or blends with weight alpha T
          bool reached = false;
          float w = 0.f;
          if (T > 0.f && b0 + base + bit < lim) {
            const float power = pair_power(q0, q1, pxf, pyf);
            if (!(power > 0.0f)) {
              const float alpha = pair_alpha(q1, power);
              if (!(alpha < 1.0f / 255.0f)) {
                reached = true;
                const float test_T = __fmul_rn(T, __fsub_rn(1.0f, alpha));
                if (test_T < 0.0001f) {
                  T = -T;
                } else {
                  w = __fmul_rn(alpha, T);
                  T = test_T;
                }
              }
            }
          }
          const unsigned rmask = __ballot_sync(FULL, reached);
          if (rmask == 0) continue;
          // exact integer sums over the block's 32 pixels (w < 2^32 in fixed point: 16-bit halves cannot overflow)
          const unsigned q = __float2uint_rn(w * CONTRIB_FIX);
          const unsigned hi = __reduce_add_sync(FULL, q >> 16), lo = __reduce_add_sync(FULL, q & 0xffffu);
          const unsigned mx = __reduce_max_sync(FULL, __float_as_uint(w));  // w >= 0: bits order like values
          if (lane == 0) {
            const int g = __float_as_int(rec[2].z);
            atomicAdd(&count[g], (unsigned long long)__popc(rmask));
            const unsigned long long s = ((unsigned long long)hi << 16) + lo;
            if (s) atomicAdd(&fixed_w[g], s);
            if (mx) atomicMax(&max_w[g], mx);
          }
        }
      }
    }
    if (__syncthreads_and(T < 0.f || b0 + CONTRIB_THREADS >= lim)) break;
  }
}

// weight[i] += fixed_w[i] 2^-32 in double, views folded in stream order
__global__ void k_contrib_fold(int P, const unsigned long long* __restrict__ fixed_w, double* __restrict__ weight) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < P && fixed_w[i]) weight[i] += (double)fixed_w[i] * (1.0 / 4294967296.0);
}

}  // namespace

// Experiment knob (GSR_RENDER_PAD=<bytes>, read once): extra dynamic shared memory per compositing CTA.  It lowers the
// number of compositing CTAs resident per SM so that CTAs of other streams' memory-bound kernels can co-reside.
static size_t render_pad() {
  static const size_t v = [] { const char* e = getenv("GSR_RENDER_PAD"); return e ? (size_t)atol(e) : (size_t)0; }();
  return v;
}
template <typename K> static void allow_pad(K kernel) {
  if (render_pad()) cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)render_pad());
}

void launch_render_fwd(int W, int H, int gx, int gy, ImageView im, BinView b, GeomView g, bool tma, float* out_color,
                       float* out_depth, float* out_median, float* out_opacity, cudaStream_t st) {
  auto kernel = tma ? k_render_fwd<true> : k_render_fwd<false>;
  allow_pad(kernel);
  kernel<<<gx * gy, FWD_THREADS, render_pad(), st>>>(W, H, gx, im, b, g.splat, out_color, out_depth, out_median, out_opacity);
}

// Pixels per lane of the compositing backward: 1 (default) or 2 (GSR_BWD_NSUB=2, read once per process).  The A/B on
// cfg 3 (1, 2, 4 and 8 pixels per lane, two occupancy targets each; not repeated on the H100) had one pixel per lane
// fastest -- fewer reductions per Gaussian do not make up for the resident warps the extra registers cost --
// so only the two-pixel variant is kept as a validated alternative (tests/test_gpu_ring_stress.py).
static int bwd_nsub() {
  static const int v = [] { const char* e = getenv("GSR_BWD_NSUB"); return (e && e[0] == '2') ? 2 : 1; }();
  return v;
}

template <int NSUB, int MINB>
static void launch_bwd(int W, int H, int gx, int gy, const float* bg, ImageView im, BinView b, GeomView g,
                       const float* dL_dpix, const float* dL_ddepth, const float* dL_dmedian, const float* dL_dopacity,
                       cudaStream_t st) {
  allow_pad(k_render_bwd<NSUB, MINB>);
  k_render_bwd<NSUB, MINB><<<gx * gy, (NBLK / NSUB) * 32 + 32, render_pad(), st>>>(W, H, gx, bg, im, b, g.splat, g.grad, dL_dpix,
                                                                       dL_ddepth, dL_dmedian, dL_dopacity);
}

void launch_render_bwd(int W, int H, int gx, int gy, const float* bg, ImageView im, BinView b, GeomView g,
                       const float* dL_dpix, const float* dL_ddepth, const float* dL_dmedian,
                       const float* dL_dopacity, cudaStream_t st) {
  if (bwd_nsub() == 2) launch_bwd<2, 4>(W, H, gx, gy, bg, im, b, g, dL_dpix, dL_ddepth, dL_dmedian, dL_dopacity, st);
  else launch_bwd<1, 4>(W, H, gx, gy, bg, im, b, g, dL_dpix, dL_ddepth, dL_dmedian, dL_dopacity, st);
}

}  // namespace gsr

using namespace gsr;

extern "C" {

int gsr_contribution(int P, int64_t R, int width, int height, char* geom_buffer, const char* binning_buffer,
                     const char* image_buffer, double* weight, int64_t* count, float* max_weight, void* stream) {
  const char* fn = "gsr_contribution";
  if (P < 0 || width <= 0 || height <= 0) return fail(fn, "P >= 0, width and height must be positive");
  const int gx = (width + TILE_X - 1) / TILE_X, gy = (height + TILE_Y - 1) / TILE_Y;
  if (gx > 65535 || gy > 65535) return fail(fn, "image too large");
  if (P == 0) return 0;
  if (!geom_buffer || !image_buffer || (R > 0 && !binning_buffer)) return fail(fn, "missing state buffers");
  if (!weight || !count || !max_weight) return fail(fn, "weight, count and max_weight are required");
  cudaStream_t st = (cudaStream_t)stream;
  GeomView g = carve_geom(aligned_base(geom_buffer), P);
  // the per-view fixed-point sums live in the backward's scratch (48 B per Gaussian), which a backward re-initialises
  unsigned long long* fixed_w = reinterpret_cast<unsigned long long*>(g.grad);
  if (!check(cudaMemsetAsync(fixed_w, 0, sizeof(unsigned long long) * (size_t)P, st), fn)) return -1;
  if (R > 0) {
    ImageView im = carve_image(aligned_base(const_cast<char*>(image_buffer)), width, height);
    BinView b = carve_binning(aligned_base(const_cast<char*>(binning_buffer)), R);
    k_render_contrib<<<gx * gy, CONTRIB_THREADS, 0, st>>>(width, height, gx, im, b, g.splat, fixed_w,
                                                          reinterpret_cast<unsigned long long*>(count),
                                                          reinterpret_cast<unsigned*>(max_weight));
  }
  k_contrib_fold<<<blocks(P, 256), 256, 0, st>>>(P, fixed_w, weight);
  return launched(fn);
}

}  // extern "C"
