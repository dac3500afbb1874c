// Two-level binning: replaces duplicateWithKeys + cub::DeviceRadixSort::SortPairs + identifyTileRanges
// ($RAST/cuda_rasterizer/rasterizer_impl.cu:70-138, 278-321).  cub-free.
//
// The reference sorts R (tile<<32 | depth bits) keys with a 6-pass LSD radix sort (~152 B of HBM traffic
// per tile instance).  The tile id is the most significant field and per-tile counts are a by-product of
// the projection kernel, so the same total order is produced with far less traffic:
//   level 1  counting sort by tile: an exclusive scan of the tile histogram gives the tile ranges directly
//            (no memset + identifyTileRanges pass); every Gaussian then scatters one 8-byte entry
//            (depth bits << 32 | gaussian index) per touched tile through per-tile write cursors.  Counters
//            and cursors are split into SUBBINS per tile so the returning atomics do not serialise on one
//            L2 address for a crowded tile;
//   level 2  each tile's segment is sorted by one CTA (MSD split into depth buckets + one warp-level bitonic
//            network per bucket) -- in shared memory when it fits, in global memory (L2-resident) otherwise --
//            and the sorted order is written as the list of Gaussian indices (the reference's point_list); the
//            render kernels gather the 48-byte splat records through it, asynchronously, only as far as the
//            tile actually gets consumed.
// Order parity: the reference's sort is stable and its emit order is ascending Gaussian index
// (rasterizer_impl.cu:98-108), so "stable by (tile, depth bits)" == total order by
// (tile, depth bits, gaussian index).  Level 2 compares whole 64-bit entries, so the result never depends on
// the (non-deterministic) arrival order of the level-1 scatter.
#include "gsr_internal.cuh"
#include <atomic>
#include <cstdlib>
#ifndef GSR_WITH_CLUSTER_SCAN
#define GSR_WITH_CLUSTER_SCAN 0
#endif
#if GSR_WITH_CLUSTER_SCAN
#include <cooperative_groups.h>
namespace cg = cooperative_groups;
#endif


namespace gsr {

namespace {

constexpr unsigned FULL = 0xffffffffu;

// ---- level 1a: tile totals + exclusive scan (one CTA; T is at most a few 10^5) --------------------
// Rounds of SCAN_TILES tiles (a 1080p image is one round).  Every global access is coalesced over consecutive tiles:
//   1. tile totals (SUBBINS counters each, all loads of a thread in flight together) -> shared memory;
//   2. ONE block scan per round: a thread scans its 8 consecutive totals in shared memory, warp / block carry;
//   3. ranges and sub-bin write cursors, from the scanned totals and a second, cache-resident read of the counters.
constexpr int SCAN_THREADS = 1024;
constexpr int SCAN_TPT = 8;
constexpr int SCAN_TILES = SCAN_THREADS * SCAN_TPT;
constexpr int SORT_CAP_SMALL_ = 6144;  // == SORT_CAP_SMALL below
__global__ void __launch_bounds__(SCAN_THREADS) k_tile_scan(ImageView im, int T, int longest_first) {
  __shared__ unsigned total[SCAN_TILES];  // tile totals, then their exclusive prefix within the round
  __shared__ unsigned warp_sums[32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned long long cap = im.hdr->capacity;
  unsigned long long carry = 0;
  for (int t0 = 0; t0 < T; t0 += SCAN_TILES) {
#pragma unroll
    for (int k = 0; k < SCAN_TPT; k++) {
      const int t = t0 + k * SCAN_THREADS + tid;
      unsigned c = 0;
      if (t < T) {
#pragma unroll
        for (int s = 0; s < SUBBINS; s++) c += im.tile_count[s * T + t];
      }
      total[k * SCAN_THREADS + tid] = c;
    }
    __syncthreads();
    // thread `tid` scans tiles [tid * SCAN_TPT, +SCAN_TPT) of the round
    unsigned v[SCAN_TPT], local = 0;
#pragma unroll
    for (int k = 0; k < SCAN_TPT; k++) { v[k] = total[tid * SCAN_TPT + k]; local += v[k]; }
    unsigned incl = local;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned u = __shfl_up_sync(FULL, incl, o); if (lane >= o) incl += u; }
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    unsigned wv = warp_sums[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned u = __shfl_up_sync(FULL, wv, o); if (lane >= o) wv += u; }
    const unsigned round_total = __shfl_sync(FULL, wv, 31);
    const unsigned before_warp = __shfl_sync(FULL, wv, max(warp - 1, 0));
    unsigned run = (warp ? before_warp : 0u) + (incl - local);
#pragma unroll
    for (int k = 0; k < SCAN_TPT; k++) {
      total[tid * SCAN_TPT + k] = run;  // exclusive prefix inside the round (own slots only: no hazard)
      run += v[k];
    }
    __syncthreads();
#pragma unroll 2
    for (int k = 0; k < SCAN_TPT; k++) {
      const int t = t0 + k * SCAN_THREADS + tid;
      if (t < T) {
        unsigned cnt[SUBBINS], c = 0;  // second read of the counters: L1 / L2 resident
#pragma unroll
        for (int s = 0; s < SUBBINS; s++) { cnt[s] = im.tile_count[s * T + t]; c += cnt[s]; }
        unsigned long long at = carry + total[k * SCAN_THREADS + tid];
        // tiles whose segment does not fit the binning capacity render nothing (pipelined-mode overflow)
        const bool fits = at + c <= cap;
        im.tile_range[t] = (c && fits) ? make_uint2((unsigned)at, (unsigned)(at + c)) : make_uint2(0u, 0u);
        if (fits && c > (unsigned)SORT_CAP_SMALL_) im.big_tiles[atomicAdd(&im.hdr->num_big, 1u)] = (unsigned)t;
#pragma unroll
        for (int s = 0; s < SUBBINS; s++) {
          im.tile_cursor[s * T + t] = fits ? (unsigned)at : 0x80000000u;  // dropped: slots fail the range test
          at += cnt[s];
        }
      }
    }
    carry += round_total;
    __syncthreads();
  }
  if (tid == 0) {
    im.hdr->num_rendered = carry;
    im.hdr->overflow = carry > cap ? 1u : 0u;
  }
  // Longest-first launch order for the one-CTA-per-tile kernels (sort, compositing): a counting sort of the tiles into
  // 64 size classes, heaviest class first.  Within a class the order is whatever the atomics give -- it only decides
  // which CTA index works on which tile, never a result.
  if (longest_first == 0) {  // raster order
    for (int t = tid; t < T; t += SCAN_THREADS) im.tile_order[t] = (uint32_t)t;
    return;
  }
  __shared__ unsigned cls_count[64], cls_start[64];
  if (tid < 64) cls_count[tid] = 0;
  __syncthreads();  // also makes this CTA's tile_range writes visible to itself
  auto size_class = [&](int t) {
    const uint2 r = im.tile_range[t];
    return 63u - min(63u, (r.y - r.x) >> 6);  // class 0: >= 4032 instances ... class 63: < 64 (incl. empty)
  };
  for (int t = tid; t < T; t += SCAN_THREADS) atomicAdd(&cls_count[size_class(t)], 1u);
  __syncthreads();
  if (tid == 0) {
    unsigned run = 0;
    for (int c = 0; c < 64; c++) { cls_start[c] = run; run += cls_count[c]; }
  }
  __syncthreads();
  for (int t = tid; t < T; t += SCAN_THREADS) {
    const unsigned pos = atomicAdd(&cls_start[size_class(t)], 1u);
    im.tile_order[longest_first == 2 ? (unsigned)T - 1u - pos : pos] = (uint32_t)t;  // 2: shortest first
  }
}

#if GSR_WITH_CLUSTER_SCAN
// ---- level 1a, cluster form: the same scan by a thread-block cluster of 8 CTAs -- EXPERIMENTAL, not in the default build
// Compiled only with -DGSR_WITH_CLUSTER_SCAN=1 (tools/build_variants.py cluster_scan) and then selected at run time with
// GSR_SCAN_CLUSTER=1.  It is faster than the single-CTA scan and passed the whole GPU suite, but with it the first
// un-fused render of tests/test_gpu_api.py::test_fused_path_with_mostly_culled_ctas_... came out slightly different
// (not reproducible on re-render) more often than without it; the cause was not found, so the validated single-CTA
// kernel stays the product path (DESIGN.md 3.5).
// The single-CTA scan is pure latency on one SM (at 1080p: 8160 tiles x 16 counters through one SM's load path,
// twice, plus a counting sort with contended shared-memory atomics).  Here every thread owns ONE tile per round (a round
// = 8 x 1024 tiles: a 1080p image is one round), its 16 counters stay in registers between the total and the cursor
// pass, the 8 CTAs exchange their round totals through distributed shared memory (one cluster barrier per round), and
// the size-class counting sort of the launch order uses warp-aggregated atomics and a cluster-wide class histogram.
// Intended outputs: those of k_tile_scan except for the (free) order of tiles inside a size class and of the crowded-tile list.
constexpr int SCAN_CLUSTER = 8;
#ifndef GSR_SCAN_CL_THREADS
#define GSR_SCAN_CL_THREADS 512
#endif
constexpr int SCAN_CL_THREADS = GSR_SCAN_CL_THREADS;  // 512: a 1080p image is two rounds; half an SM's threads per CTA,
                                                      // so the cluster finds room next to other views' kernels sooner
static_assert(SCAN_CL_THREADS % 64 == 0 && SCAN_CL_THREADS >= 64 && SCAN_CL_THREADS <= 1024, "cluster scan CTA size");
__global__ void __cluster_dims__(SCAN_CLUSTER, 1, 1) __launch_bounds__(SCAN_CL_THREADS)
k_tile_scan_cluster(ImageView im, int T, int longest_first) {
  cg::cluster_group cluster = cg::this_cluster();
  const unsigned rank = cluster.block_rank();
  __shared__ unsigned warp_sums[32];
  __shared__ unsigned cta_total[2];  // this CTA's total of the round, double-buffered by round parity
  __shared__ unsigned cls_count[64], cls_start[64];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned long long cap = im.hdr->capacity;
  unsigned long long carry = 0;  // tiles of earlier rounds (the same value in every CTA)
  constexpr int ROUND = SCAN_CLUSTER * SCAN_CL_THREADS;
  int round = 0;
  for (int t0 = 0; t0 < T; t0 += ROUND, round++) {
    const int t = t0 + (int)rank * SCAN_CL_THREADS + tid;
    unsigned cnt[SUBBINS], c = 0;
#pragma unroll
    for (int s = 0; s < SUBBINS; s++) { cnt[s] = t < T ? im.tile_count[s * T + t] : 0u; c += cnt[s]; }
    unsigned incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned u = __shfl_up_sync(FULL, incl, o); if (lane >= o) incl += u; }
    __syncthreads();  // warp_sums of the previous round are consumed
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    unsigned wv = lane < SCAN_CL_THREADS / 32 ? warp_sums[lane] : 0u;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned u = __shfl_up_sync(FULL, wv, o); if (lane >= o) wv += u; }
    const unsigned my_total = __shfl_sync(FULL, wv, 31);
    const unsigned before_warp = __shfl_sync(FULL, wv, max(warp - 1, 0));
    const unsigned excl = (warp ? before_warp : 0u) + (incl - c);  // exclusive prefix inside this CTA's tiles of the round
    if (tid == 0) cta_total[round & 1] = my_total;
    cluster.sync();  // every CTA's total of this round is published
    unsigned before = 0, all = 0;
#pragma unroll
    for (unsigned r = 0; r < (unsigned)SCAN_CLUSTER; r++) {
      const unsigned v = *cluster.map_shared_rank(&cta_total[round & 1], r);
      before += r < rank ? v : 0u;
      all += v;
    }
    if (t < T) {
      unsigned long long at = carry + before + excl;
      // tiles whose segment does not fit the binning capacity render nothing (pipelined-mode overflow)
      const bool fits = at + c <= cap;
      im.tile_range[t] = (c && fits) ? make_uint2((unsigned)at, (unsigned)(at + c)) : make_uint2(0u, 0u);
      if (fits && c > (unsigned)SORT_CAP_SMALL_) im.big_tiles[atomicAdd(&im.hdr->num_big, 1u)] = (unsigned)t;
#pragma unroll
      for (int s = 0; s < SUBBINS; s++) {
        im.tile_cursor[s * T + t] = fits ? (unsigned)at : 0x80000000u;  // dropped: slots fail the range test
        at += cnt[s];
      }
    }
    carry += all;
  }
  if (rank == 0 && tid == 0) {
    im.hdr->num_rendered = carry;
    im.hdr->overflow = carry > cap ? 1u : 0u;
  }
  // launch order of the one-CTA-per-tile kernels: see k_tile_scan
  if (longest_first == 0) {  // raster order
    for (int t0 = 0; t0 < T; t0 += ROUND) {
      const int t = t0 + (int)rank * SCAN_CL_THREADS + tid;
      if (t < T) im.tile_order[t] = (uint32_t)t;
    }
    cluster.sync();  // a CTA must not exit while another one may still read its round total
    return;
  }
  if (tid < 64) cls_count[tid] = 0;
  __syncthreads();  // also makes this CTA's tile_range writes visible to itself
  auto size_class = [&](int t) {
    const uint2 r = im.tile_range[t];
    return 63u - min(63u, (r.y - r.x) >> 6);  // class 0: >= 4032 instances ... class 63: < 64 (incl. empty)
  };
  // one shared-memory atomic per (warp, class): lanes of the same class elect a leader
  auto claim = [&](unsigned* counters, unsigned cls, bool active) -> unsigned {
    const unsigned peers = __match_any_sync(FULL, active ? cls : 0xffffffffu);
    const int leader = __ffs(peers) - 1;
    unsigned base = 0;
    if (active && lane == leader) base = atomicAdd(&counters[cls], (unsigned)__popc(peers));
    base = __shfl_sync(FULL, base, leader);
    return base + (unsigned)__popc(peers & ((1u << lane) - 1u));
  };
  for (int t0 = 0; t0 < T; t0 += ROUND) {
    const int t = t0 + (int)rank * SCAN_CL_THREADS + tid;
    claim(cls_count, t < T ? size_class(t) : 0u, t < T);
  }
  cluster.sync();  // every CTA's class histogram is complete
  if (tid < 64) {
    unsigned tot = 0, mine = 0;
#pragma unroll
    for (unsigned r = 0; r < (unsigned)SCAN_CLUSTER; r++) {
      const unsigned v = *cluster.map_shared_rank(&cls_count[tid], r);
      mine += r < rank ? v : 0u;
      tot += v;
    }
    // exclusive prefix of the cluster-wide class totals over the 64 classes (two warps)
    unsigned incl = tot;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned u = __shfl_up_sync(FULL, incl, o); if (lane >= o) incl += u; }
    if (tid == 31) warp_sums[0] = incl;
    asm volatile("bar.sync 1, 64;" ::: "memory");
    cls_start[tid] = (tid >= 32 ? warp_sums[0] : 0u) + (incl - tot) + mine;
  }
  cluster.sync();  // the remote histograms have been read (a CTA may exit), and cls_start is visible to this CTA
  for (int t0 = 0; t0 < T; t0 += ROUND) {
    const int t = t0 + (int)rank * SCAN_CL_THREADS + tid;
    const unsigned pos = claim(cls_start, t < T ? size_class(t) : 0u, t < T);
    if (t < T) im.tile_order[longest_first == 2 ? (unsigned)T - 1u - pos : pos] = (uint32_t)t;  // 2: shortest first
  }
}
#endif  // GSR_WITH_CLUSTER_SCAN

// ---- level 1b: scatter one entry per (Gaussian, touched tile) ------------------------------------
#ifndef GSR_SCATTER_THREADS
#define GSR_SCATTER_THREADS 256
#endif
constexpr int SCATTER_THREADS = GSR_SCATTER_THREADS;
__global__ void __launch_bounds__(SCATTER_THREADS) k_scatter(int P, int gx, int T, GeomView g, ImageView im, BinView b) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  int x0 = 0, y0 = 0, x1 = 0, y1 = 0;
  unsigned depth_bits = 0, mask = 0;
  if (idx < P) {
    const uint2 rc = g.rect[idx];
    mask = g.tile_mask[idx];
    unpack_rect(rc, x0, y0, x1, y1);
    // (the record of a culled Gaussian is never written: do not touch it)
    if (x1 > x0) depth_bits = __float_as_uint(reinterpret_cast<const float*>(g.splat + (size_t)idx * SPLAT_F4 + 1)[2]);
  }
  const int w = x1 - x0, n = w * (y1 - y0);
  const unsigned lane = threadIdx.x & 31;
  constexpr int kBig = 32;  // == kBigRect of the projection kernel: larger rects are binned in full
  // cursors of tiles that were dropped for capacity start at DROPPED, so their slots fail the range test
  const unsigned long long cap = im.hdr->capacity;
  const unsigned limit = cap < 0x80000000ull ? (unsigned)cap : 0x80000000u;
  auto put = [&](int tile, unsigned dbits, int gidx) {
    const unsigned slot = atomicAdd(&im.tile_cursor[subbin_of(gidx) * T + tile], 1u);
    if (slot < limit) b.ents[slot] = ((unsigned long long)dbits << 32) | (unsigned)gidx;
  };
  if (n > 0 && n <= kBig) {
    // eight binned tiles at a time: the returning atomics are independent and overlap their L2 round trips (a typical
    // splat keeps 2-4 of its tiles, so most threads need a single round)
    const unsigned long long key = ((unsigned long long)depth_bits << 32) | (unsigned)idx;
    unsigned* cur = im.tile_cursor + subbin_of(idx) * T;
    constexpr int kFlight = 8;
    while (mask) {
      unsigned slot[kFlight];
#pragma unroll
      for (int k = 0; k < kFlight; k++) {
        slot[k] = 0xffffffffu;
        if (mask) {
          const int i = __ffs(mask) - 1;
          mask &= mask - 1;
          slot[k] = atomicAdd(cur + (y0 + i / w) * gx + x0 + i % w, 1u);
        }
      }
#pragma unroll
      for (int k = 0; k < kFlight; k++)
        if (slot[k] < limit) b.ents[slot[k]] = key;
    }
  }
  // a splat covering many tiles is walked by the whole warp (see for_each_tile in gsr_internal.cuh)
  unsigned big = __ballot_sync(FULL, n > kBig);
  while (big) {
    const int src = __ffs(big) - 1;
    big &= big - 1;
    const int bx0 = __shfl_sync(FULL, x0, src), by0 = __shfl_sync(FULL, y0, src);
    const int bw = __shfl_sync(FULL, w, src), bn = __shfl_sync(FULL, n, src);
    const unsigned sd = __shfl_sync(FULL, depth_bits, src);
    const int sidx = __shfl_sync(FULL, idx, src);
    for (int i = lane; i < bn; i += 32) put((by0 + i / bw) * gx + bx0 + i % bw, sd, sidx);
  }
}

// ---- level 2: per-tile sort + slab gather ---------------------------------------------------------
// One CTA per tile.  An MSD split maps the depth keys linearly from the tile's own [min, max] onto NB depth
// buckets (shared-memory atomics: the split need not be stable), then every bucket -- about 8 entries -- is
// sorted by one warp with a shuffle bitonic network on the full 64-bit
// entry (depth bits << 32 | gaussian index).  Comparing the whole entry yields the reference's order
// (stable by depth == ties in ascending Gaussian index) with no dependence on the scatter's arrival order.
constexpr int SORT_THREADS = 512;
#ifndef GSR_SORT_THREADS_TINY
#define GSR_SORT_THREADS_TINY 128
#endif
#ifndef GSR_SORT_CAP_TINY
#define GSR_SORT_CAP_TINY 2048
#endif
constexpr int SORT_THREADS_TINY = GSR_SORT_THREADS_TINY;  // CTA size of the tier that owns the tiles with <= SORT_CAP_TINY instances
constexpr int SORT_CAP_TINY = GSR_SORT_CAP_TINY;
constexpr int SORT_WARPS = SORT_THREADS / 32;
// Four launches cover every tile: 128-thread CTAs (one per tile, ~13 per SM) for tiles up to SORT_CAP_TINY entries --
// most tiles of a view, where a 512-thread CTA would mostly idle through the passes --, 512-thread CTAs (one per tile,
// 4 CTAs/SM) up to SORT_CAP_SMALL, a two-CTAs-per-SM kernel up to SORT_CAP_MID and a one-CTA-per-SM kernel with
// almost all of the SM's shared memory for the most crowded ones; only tiles beyond SORT_CAP_BIG entries fall back
// to sorting in global memory (L2-resident scratch).  The two crowded tiers take their tiles from the compact list
// the scan produced through an atomic ticket, so a CTA that drew a 25k-entry tile does not hold up a queue of others.
constexpr int SORT_CAP_SMALL = 6144;   // 48 KB: four CTAs per SM
constexpr int SORT_CAP_MID = 12288;    // 96 KB: two CTAs per SM
static_assert(SORT_CAP_SMALL == SORT_CAP_SMALL_, "scan and sort disagree on the small-tier capacity");
constexpr int SORT_CAP_BIG = 26624;    // 208 KB (+ 16 KB of bucket counters)
typedef unsigned long long u64;

// ascending bitonic sort of one key per lane (unused lanes hold ~0ull)
__device__ __forceinline__ u64 warp_sort32(u64 key, unsigned lane) {
#pragma unroll
  for (unsigned k = 2; k <= 32; k <<= 1) {
#pragma unroll
    for (unsigned j = k >> 1; j > 0; j >>= 1) {
      const u64 other = __shfl_xor_sync(FULL, key, j);
      const bool up = (lane & k) == 0 || k == 32;
      const bool lower = (lane & j) == 0;
      const u64 mn = key < other ? key : other, mx = key < other ? other : key;
      key = (lower == up) ? mn : mx;
    }
  }
  return key;
}

// one warp sorts k[0,m) in place (shared or global memory), m > 32: "all ascending" bitonic network, where
// indices >= m behave as +inf (such pairs never swap and are skipped)
__device__ __forceinline__ void warp_sort_mem(u64* k, unsigned m, unsigned lane) {
  unsigned npad = 64;
  while (npad < m) npad <<= 1;
  const unsigned half = npad >> 1;
  for (unsigned blk = 2; blk <= npad; blk <<= 1) {
    const unsigned hb = blk >> 1;
    for (unsigned t = lane; t < half; t += 32) {
      const unsigned base = (t / hb) * blk, off = t % hb, i = base + off, p = base + blk - 1 - off;
      if (p < m) { const u64 a = k[i], c = k[p]; if (a > c) { k[i] = c; k[p] = a; } }
    }
    __syncwarp();
    for (unsigned j = blk >> 2; j > 0; j >>= 1) {
      for (unsigned t = lane; t < half; t += 32) {
        const unsigned i = 2 * j * (t / j) + (t % j), p = i + j;
        if (p < m) { const u64 a = k[i], c = k[p]; if (a > c) { k[i] = c; k[p] = a; } }
      }
      __syncwarp();
    }
  }
}

// r += (o < k): one predicated add (the compiler's own form is an add plus a predicated move on the dependent chain)
__device__ __forceinline__ void count_if_less(unsigned& r, u64 o, u64 k) {
  asm("{ .reg .pred p; setp.lt.u64 p, %1, %2; @p add.u32 %0, %0, 1; }" : "+r"(r) : "l"(o), "l"(k));
}

template <int NB> struct SortShared {
  unsigned cnt[NB];        // bucket sizes, then running cursors of the split
  unsigned start[NB + 1];  // exclusive prefix of the bucket sizes
  alignas(16) unsigned wsum[SORT_WARPS];  // own 16-byte slots: the compiler reads them with vector loads
  unsigned dmin, dmax;
};

// CAP: entries held in shared memory; this launch owns the tiles with MIN_N < n <= MAX_N entries (MAX_N = 0: no upper
// bound; beyond CAP the tile is sorted in the global scratch); NB: depth buckets of the MSD split; TIER: ticket index.
// DIRECT: one CTA per tile (blockIdx -> tile_order); otherwise CTAs draw tickets into the list of crowded tiles.
// THREADS: CTA size (<= SORT_THREADS).
template <int CAP, int MIN_N, int MAX_N, int NB, int TIER, bool DIRECT, int THREADS>
__global__ void __launch_bounds__(THREADS) k_tile_sort(GeomView g, ImageView im, BinView b) {
  constexpr int WARPS = THREADS / 32;
  extern __shared__ __align__(16) u64 sort_smem[];
  __shared__ SortShared<NB> sh;
  __shared__ unsigned sh_work;
  const unsigned tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // small launch: one CTA per tile.  crowded launches: CTAs draw tiles from the compact list of crowded tiles.
  const unsigned num_work = DIRECT ? gridDim.x : im.hdr->num_big;
  for (unsigned work = blockIdx.x;; work += gridDim.x) {
  if (!DIRECT) {
    __syncthreads();  // everybody is done with the previous tile (and with sh_work)
    if (tid == 0) sh_work = atomicAdd(&im.hdr->ticket[TIER], 1u);
    __syncthreads();
    work = sh_work;
  }
  if (work >= num_work) break;
  const unsigned tile = DIRECT ? im.tile_order[work] : im.big_tiles[work];
  const uint2 range = im.tile_range[tile];
  const unsigned n = range.y - range.x;
  if (n <= (unsigned)MIN_N || (MAX_N != 0 && n > (unsigned)MAX_N)) continue;  // another launch owns this tile
  __syncthreads();  // shared memory of the previous tile is free
  u64* seg = b.ents + range.x;
  uint32_t* out = b.point_list + range.x;
  const u64* sorted;

  if (n <= 32) {
    // a single warp sorts the whole tile in registers
    if (warp == 0) {
      const u64 key = warp_sort32(lane < n ? seg[lane] : ~0ull, lane);
      if (lane < n) sort_smem[lane] = key;
    }
    __syncthreads();
    sorted = sort_smem;
  } else {
    const bool in_smem = n <= (unsigned)CAP;
    // A: unsorted input, B: bucketed + sorted output (shared memory, or the L2-resident scratch segment for a
    // tile with more instances than fit).
    const u64* A = seg;
    u64* B = in_smem ? sort_smem : b.ents2 + range.x;
    for (unsigned i = tid; i < NB; i += THREADS) sh.cnt[i] = 0;
    if (tid == 0) { sh.dmin = 0xffffffffu; sh.dmax = 0u; }
    __syncthreads();
    // bucket = linear map of the depth bits from the tile's own [min, max] onto [0, NB): monotone in depth, and
    // balanced even when the tile's depths span several binades but crowd into one of them
    unsigned lo = 0xffffffffu, hi = 0u;
    for (unsigned i = tid; i < n; i += THREADS) { const unsigned d = (unsigned)(A[i] >> 32); lo = min(lo, d); hi = max(hi, d); }
    lo = __reduce_min_sync(FULL, lo); hi = __reduce_max_sync(FULL, hi);
    if (lane == 0) { atomicMin(&sh.dmin, lo); atomicMax(&sh.dmax, hi); }
    __syncthreads();
    const unsigned dmin = sh.dmin, span = sh.dmax - dmin;
    // bucket = floor((d - dmin) * NB / (span + 1)) via a 32-bit fixed-point reciprocal (span >= NB here), or the
    // identity when the tile's keys span fewer values than there are buckets
    // one warp sorts one bucket: aim at ~24 entries per bucket (full lanes, rare spill beyond 64)
    const unsigned nb = min((unsigned)NB, max(8u, n / 24u));
    const bool direct = span < nb;
    const unsigned mult = direct ? 0u : (unsigned)(((u64)nb << 32) / ((u64)span + 1ull));
    auto bucket = [=](u64 key) {
      const unsigned d = (unsigned)(key >> 32) - dmin;
      return direct ? d : __umulhi(d, mult);
    };
    for (unsigned i = tid; i < n; i += THREADS) atomicAdd(&sh.cnt[bucket(A[i])], 1u);
    __syncthreads();
    {  // exclusive scan of the NB bucket sizes: NB / THREADS consecutive buckets per thread
      constexpr int PER = (NB + THREADS - 1) / THREADS;
      unsigned c[PER], local = 0;
#pragma unroll
      for (int k = 0; k < PER; k++) { const unsigned i = tid * PER + k; c[k] = i < NB ? sh.cnt[i] : 0u; local += c[k]; }
      unsigned v = local;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const unsigned u = __shfl_up_sync(FULL, v, o); if (lane >= o) v += u; }
      if (lane == 31) sh.wsum[warp] = v;
      __syncthreads();
      unsigned run = v - local;
#pragma unroll
      for (int w = 0; w < WARPS; w++) run += (w < (int)warp) ? sh.wsum[w] : 0u;
#pragma unroll
      for (int k = 0; k < PER; k++) {
        const unsigned i = tid * PER + k;
        if (i < NB) { sh.start[i] = run; sh.cnt[i] = run; }
        run += c[k];
      }
      if (tid == THREADS - 1) sh.start[NB] = run;
    }
    __syncthreads();
    for (unsigned i = tid; i < n; i += THREADS) {
      const u64 key = A[i];
      B[atomicAdd(&sh.cnt[bucket(key)], 1u)] = key;
    }
    __syncthreads();
    for (unsigned bk = warp; bk < nb; bk += WARPS) {
      const unsigned s0 = sh.start[bk], m = sh.start[bk + 1] - s0;
      if (m <= 1) continue;
      if (m <= 32) {
        // rank sort, one entry per lane: entries are distinct 64-bit values, so an entry's position is the number
        // of smaller ones (m broadcast reads + compares: cheaper than a bitonic network for the ~24-entry buckets
        // the split aims at)
        const u64 k0 = lane < m ? B[s0 + lane] : ~0ull;
        unsigned r0 = 0;
#pragma unroll 8
        for (unsigned j = 0; j < m; j++) count_if_less(r0, B[s0 + j], k0);
        __syncwarp();
        if (lane < m) B[s0 + r0] = k0;
        __syncwarp();
      } else if (m <= 64) {
        // the same with two entries per lane
        const u64 k0 = B[s0 + lane];
        const u64 k1 = lane + 32 < m ? B[s0 + 32 + lane] : ~0ull;
        unsigned r0 = 0, r1 = 0;
#pragma unroll 4
        for (unsigned j = 0; j < m; j++) {
          const u64 o = B[s0 + j];
          count_if_less(r0, o, k0);
          count_if_less(r1, o, k1);
        }
        __syncwarp();
        if (lane < m) B[s0 + r0] = k0;
        if (lane + 32 < m) B[s0 + r1] = k1;
        __syncwarp();
      } else {
        warp_sort_mem(B + s0, m, lane);
      }
    }
    __syncthreads();
    sorted = B;
  }
  // the sorted order, as Gaussian indices (what the render kernels walk)
  for (unsigned i = tid; i < n; i += THREADS) out[i] = (uint32_t)sorted[i];
  }
}

}  // namespace

// GSR_TILE_ORDER=0 (read once per process): one-CTA-per-tile kernels take their tiles in raster order instead of
// longest-first (the A/B of DESIGN.md 3.4)
static std::atomic<int> g_tile_order{-1};  // gsr_set_tile_order; < 0: the default below
int set_tile_order(int mode) { return g_tile_order.exchange(mode > 2 ? -1 : mode); }
static int tile_order_mode() {  // 0 raster, 1 longest first (default), 2 shortest first
  static const int dflt = [] { const char* e = getenv("GSR_TILE_ORDER"); return (e && e[0] >= '0' && e[0] <= '2') ? e[0] - '0' : 1; }();
  const int m = g_tile_order.load();
  return m >= 0 ? m : dflt;
}
void launch_tile_scan(ImageView im, int T, cudaStream_t st) {
#if GSR_WITH_CLUSTER_SCAN
  // experimental builds only: GSR_SCAN_CLUSTER=1 (read once per process) selects the 8-CTA cluster form
  static const bool cluster = [] { const char* e = getenv("GSR_SCAN_CLUSTER"); return e && e[0] == '1'; }();
  if (cluster) {
    launch_high_priority(k_tile_scan_cluster, dim3(SCAN_CLUSTER), dim3(SCAN_CL_THREADS), 0, st, im, T, tile_order_mode());
    return;
  }
#endif
  launch_high_priority(k_tile_scan, dim3(1), dim3(SCAN_THREADS), 0, st, im, T, tile_order_mode());
}

void launch_scatter(int P, int gx, int T, GeomView g, ImageView im, BinView b, cudaStream_t st) {
  launch_high_priority(k_scatter, dim3((P + SCATTER_THREADS - 1) / SCATTER_THREADS), dim3(SCATTER_THREADS), 0, st, P, gx, T, g, im, b);
}

void launch_tile_sort(int T, GeomView g, ImageView im, BinView b, cudaStream_t st) {
  // four launches, each owning a size class: tiny tiles (most of them: small CTAs, many per SM), tiles that fit 48 KB of
  // shared memory, and the two crowded tiers drawn from the list the scan compiles
  auto tiny = k_tile_sort<SORT_CAP_TINY, 0, SORT_CAP_TINY, SORT_CAP_TINY / 16, 0, true, SORT_THREADS_TINY>;
  auto small = k_tile_sort<SORT_CAP_SMALL, SORT_CAP_TINY, SORT_CAP_SMALL, 512, 0, true, SORT_THREADS>;
  auto mid = k_tile_sort<SORT_CAP_MID, SORT_CAP_SMALL, SORT_CAP_MID, 512, 0, false, SORT_THREADS>;
  auto big = k_tile_sort<SORT_CAP_BIG, SORT_CAP_MID, 0, 2048, 1, false, SORT_THREADS>;
  constexpr int smem_tiny = SORT_CAP_TINY * 8, smem_small = SORT_CAP_SMALL * 8, smem_mid = SORT_CAP_MID * 8,
                smem_big = SORT_CAP_BIG * 8;
  const DeviceInfo& di = device_info();
  if (!di.sort_attr_set) {  // once per device
    cudaFuncSetAttribute(small, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_small);
    cudaFuncSetAttribute(mid, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_mid);
    cudaFuncSetAttribute(big, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_big);
    di.sort_attr_set = true;
  }
  launch_high_priority(tiny, dim3(T), dim3(SORT_THREADS_TINY), smem_tiny, st, g, im, b);
  launch_high_priority(small, dim3(T), dim3(SORT_THREADS), smem_small, st, g, im, b);
  launch_high_priority(mid, dim3(2 * di.sm_count), dim3(SORT_THREADS), smem_mid, st, g, im, b);  // two CTAs per SM draw the 6k-12k tiles
  launch_high_priority(big, dim3(di.sm_count), dim3(SORT_THREADS), smem_big, st, g, im, b);      // one CTA per SM draws the rest
}

}  // namespace gsr
