// Rank-normalised split-R̂, bulk ESS and tail ESS (blackjax/diagnostics.py:92-155, 341-522; Vehtari et al. 2021) over a
// device-resident history [T, C, D], entry points of include/bjx.h.
//
// The history is split into 2C chains of h = T / 2 draws; draw s of split chain k has pooled index j = k * h + s, and
// each dimension's n = 2C * h pooled draws are ranked with ties broken by j (the stable argsort of _rank_normalize).
// Dimensions are processed Dc at a time, Dc set by the scratch buffer.  Per chunk:
//   k_rank_keys       history -> segment-major [Dc][n] pairs (order-preserving key << 32 | j), transposed in shared memory;
//                     the fold pass keys |x - median| the same way
//   segmented LSD radix sort over the 32 key bits, 4 passes of 8 bits, stable, so the sorted pairs are in rank order:
//     n <= kTile      k_rank_sort_tile, one CTA sorts a whole segment in shared memory
//     n >  kTile      per pass k_rank_hist (digit counts per tile), k_rank_scan (per digit over tiles) and k_rank_scatter
//                     (stable tile-local ranking, then the digit runs written out in order); grids (tiles, Dc)
//   k_rank_scores     Blom score of every rank, scattered to its split position [h, 2C, Dc]; the order statistics of the
//                     median and the two quantiles and the NaN flag
//   k_rank_indicator  1[x <= q_lo], then 1[x >= q_hi], into the same [h, 2C, Dc] buffer
// then the existing launch_rhat / launch_ess on [h, 2C, Dc] and k_rank_finish (max, min, NaN columns).
#include <math.h>

#include <string>

#include "../../include/bjx.h"
#include "bjx_handle.h"
#include "bjx_internal.h"

using namespace bjx;

namespace {

constexpr int kTile = 4096;                 // pairs per CTA of the sort
constexpr int kSortThreads = 512;
constexpr int kSortWarps = kSortThreads / 32;
constexpr int kItems = kTile / kSortThreads;  // per thread; warp w owns the kTile / kSortWarps consecutive pairs from w
constexpr int kWarpSpan = kTile / kSortWarps;
constexpr int kStats = 8;                   // per column: the 6 order statistics, the NaN flag, padding
constexpr unsigned kNanKey = 0xFFC00000u;   // key of every NaN: above +inf (0xFF800000)
typedef unsigned long long u64;

// the order statistics the score pass extracts: positions in the sorted column, and the lerp fractions of the quantiles
struct StatPos {
  long long pos[6];  // median a, b; q_lo a, b; q_hi a, b
  double t_lo, t_hi;
};

// Order-preserving image of a float's bits: -0 -> +0 and every NaN -> one positive quiet NaN, then the sign flip.
__device__ __forceinline__ unsigned float_key(float x) {
  unsigned u = __float_as_uint(x);
  if (x == 0.0f) u = 0u;
  if (x != x) u = 0x7FC00000u;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ unsigned digit_of(u64 v, int shift) { return (unsigned)(v >> (32 + shift)) & 255u; }

// numpy's "linear" quantile between the order statistics a <= b at fraction t, in float64
__device__ __forceinline__ double lerp_quantile(float a, float b, double t) {
  if (a == b) return (double)a;
  const double da = a, db = b, diff = db - da;
  return t >= 0.5 ? db - diff * (1.0 - t) : da + diff * t;
}
__device__ __forceinline__ float column_median(const float* st) { return __fmul_rn(__fadd_rn(st[0], st[1]), 0.5f); }

// ---- key build ----------------------------------------------------------------------------------------------------
// grid (2C * ceil(h / 32), ceil(Dc / 32)), block (32, 8): a 32-draw x 32-dim tile of split chain k, read along D and
// written along j.  folded: the key of |x - median| with the column's median from the bulk statistics.
__global__ void k_rank_keys(int h, int C, int D, int d0, int Dc, long long n, const float* __restrict__ hist,
                            const float* __restrict__ stats, u64* __restrict__ pairs) {
  __shared__ float tile[32][33];
  const int sblocks = (h + 31) / 32;
  const int k = blockIdx.x / sblocks, s0 = (blockIdx.x % sblocks) * 32;
  const int c = k % C, toff = k >= C ? h : 0;
  const int dl0 = blockIdx.y * 32;
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int s = s0 + r, dl = dl0 + threadIdx.x;
    if (s < h && dl < Dc) tile[r][threadIdx.x] = hist[((size_t)(s + toff) * C + c) * D + d0 + dl];
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int dl = dl0 + r, s = s0 + threadIdx.x;
    if (s >= h || dl >= Dc) continue;
    float x = tile[threadIdx.x][r];
    if (stats) x = fabsf(__fsub_rn(x, column_median(stats + (size_t)dl * kStats)));
    const unsigned j = (unsigned)k * (unsigned)h + (unsigned)s;
    pairs[(size_t)dl * n + j] = ((u64)float_key(x) << 32) | j;
  }
}

// ---- the CTA's stable ranking of one tile by one 8-bit digit ----------------------------------------------------------
struct SortSmem {
  u64 v[kTile];
  unsigned cnt[256 * kSortWarps];  // digit-major (digit, warp): counts, then their exclusive prefix over the tile
  unsigned wsum[kSortWarps];
  unsigned base[256];               // k_rank_scatter: output offset of each digit's run, less its start in the tile
};

// Exclusive prefix sum in place over cnt (kItems consecutive entries per thread).
__device__ __forceinline__ void block_scan_cnt(SortSmem& sm) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned loc[kItems], sum = 0;
#pragma unroll
  for (int i = 0; i < kItems; ++i) {
    loc[i] = sum;
    sum += sm.cnt[threadIdx.x * kItems + i];
  }
  unsigned inc = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned y = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += y;
  }
  if (lane == 31) sm.wsum[warp] = inc;
  __syncthreads();
  unsigned wbase = 0;
  for (int w = 0; w < warp; ++w) wbase += sm.wsum[w];
  const unsigned ex = wbase + inc - sum;
#pragma unroll
  for (int i = 0; i < kItems; ++i) sm.cnt[threadIdx.x * kItems + i] = ex + loc[i];
}

// Item i of this thread is tile element warp * kWarpSpan + i * 32 + lane (valid below count).  On return pos[i] is its
// place in the tile ordered stably by digit, and cnt[d * kSortWarps] is where digit d's run starts.
__device__ __forceinline__ void tile_rank(SortSmem& sm, const u64 (&it)[kItems], int count, int shift,
                                          unsigned (&pos)[kItems]) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned lt = (1u << lane) - 1u;
#pragma unroll
  for (int i = 0; i < kItems; ++i) sm.cnt[threadIdx.x * kItems + i] = 0u;
  __syncthreads();
#pragma unroll
  for (int i = 0; i < kItems; ++i) {
    const bool ok = warp * kWarpSpan + i * 32 + lane < count;
    const unsigned d = ok ? digit_of(it[i], shift) : 256u;
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    unsigned before = 0;
    if (ok) before = sm.cnt[d * kSortWarps + warp];
    __syncwarp();
    if (ok && (peers & lt) == 0) sm.cnt[d * kSortWarps + warp] = before + __popc(peers);
    __syncwarp();
    pos[i] = before + __popc(peers & lt);
  }
  __syncthreads();
  block_scan_cnt(sm);
  __syncthreads();
#pragma unroll
  for (int i = 0; i < kItems; ++i) {
    const bool ok = warp * kWarpSpan + i * 32 + lane < count;
    if (ok) pos[i] += sm.cnt[digit_of(it[i], shift) * kSortWarps + warp];
  }
}

__device__ __forceinline__ void load_items(const u64* src, int count, u64 (&it)[kItems]) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < kItems; ++i) {
    const int e = warp * kWarpSpan + i * 32 + lane;
    it[i] = e < count ? src[e] : 0ull;
  }
}

// A whole segment (n <= kTile) per CTA, sorted in place: grid Dc.
__global__ void __launch_bounds__(kSortThreads) k_rank_sort_tile(int n, u64* __restrict__ pairs) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  SortSmem& sm = *reinterpret_cast<SortSmem*>(smem_raw);
  u64* seg = pairs + (size_t)blockIdx.x * n;
  u64 it[kItems];
  unsigned pos[kItems];
  load_items(seg, n, it);
  for (int shift = 0; shift < 32; shift += 8) {
    tile_rank(sm, it, n, shift, pos);
    const int base = (threadIdx.x >> 5) * kWarpSpan + (threadIdx.x & 31);
#pragma unroll
    for (int i = 0; i < kItems; ++i)
      if (base + i * 32 < n) sm.v[pos[i]] = it[i];
    __syncthreads();
    load_items(sm.v, n, it);
    __syncthreads();
  }
  for (int e = threadIdx.x; e < n; e += kSortThreads) seg[e] = sm.v[e];
}

// Digit counts of every (segment, tile): hist[(seg * 256 + digit) * tiles + tile].  grid (tiles, Dc).
__global__ void __launch_bounds__(kSortThreads) k_rank_hist(long long n, int tiles, int shift, const u64* __restrict__ src,
                                                            unsigned* __restrict__ hist) {
  __shared__ unsigned cnt[256];
  if (threadIdx.x < 256) cnt[threadIdx.x] = 0u;
  __syncthreads();
  const long long t0 = (long long)blockIdx.x * kTile;
  const int count = (int)min((long long)kTile, n - t0);
  const u64* seg = src + (size_t)blockIdx.y * n + t0;
  for (int e = threadIdx.x; e < count; e += kSortThreads) atomicAdd(&cnt[digit_of(seg[e], shift)], 1u);
  __syncthreads();
  if (threadIdx.x < 256) hist[((size_t)blockIdx.y * 256 + threadIdx.x) * tiles + blockIdx.x] = cnt[threadIdx.x];
}

// Exclusive prefix over the tiles of one (digit, segment) in place, and the digit's total.  grid (256, Dc), 256 threads.
__global__ void __launch_bounds__(256) k_rank_scan(int tiles, unsigned* __restrict__ hist, unsigned* __restrict__ total) {
  __shared__ unsigned wsum[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned* row = hist + ((size_t)blockIdx.y * 256 + blockIdx.x) * tiles;
  unsigned carry = 0;
  for (int b = 0; b < tiles; b += 256 * 4) {
    unsigned v[4], sum = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int e = b + threadIdx.x * 4 + i;
      v[i] = e < tiles ? row[e] : 0u;
      sum += v[i];
    }
    unsigned inc = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned y = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += y;
    }
    if (lane == 31) wsum[warp] = inc;
    __syncthreads();
    unsigned wbase = 0, all = 0;
    for (int w = 0; w < 8; ++w) {
      wbase += w < warp ? wsum[w] : 0u;
      all += wsum[w];
    }
    unsigned run = carry + wbase + inc - sum;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int e = b + threadIdx.x * 4 + i;
      if (e < tiles) row[e] = run;
      run += v[i];
    }
    carry += all;
    __syncthreads();
  }
  if (threadIdx.x == 0) total[(size_t)blockIdx.y * 256 + blockIdx.x] = carry;
}

// One stable pass of a tile: rank by digit in shared memory, then each digit's run written to its place in dst.
// grid (tiles, Dc).
__global__ void __launch_bounds__(kSortThreads, 1) k_rank_scatter(long long n, int tiles, int shift, const u64* __restrict__ src,
                                                               const unsigned* __restrict__ hist,
                                                               const unsigned* __restrict__ total, u64* __restrict__ dst) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  SortSmem& sm = *reinterpret_cast<SortSmem*>(smem_raw);
  const long long t0 = (long long)blockIdx.x * kTile;
  const int count = (int)min((long long)kTile, n - t0);
  const size_t seg = (size_t)blockIdx.y * n;
  u64 it[kItems];
  unsigned pos[kItems];
  load_items(src + seg + t0, count, it);
  tile_rank(sm, it, count, shift, pos);
  const int first = (threadIdx.x >> 5) * kWarpSpan + (threadIdx.x & 31);
#pragma unroll
  for (int i = 0; i < kItems; ++i)
    if (first + i * 32 < count) sm.v[pos[i]] = it[i];
  // the segment's digit runs start at the exclusive prefix of the digit totals (first 8 warps, one digit per thread)
  if (threadIdx.x < 256) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned tot = total[(size_t)blockIdx.y * 256 + threadIdx.x];
    unsigned inc = tot;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned y = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += y;
    }
    if (lane == 31) sm.wsum[warp] = inc;
    sm.base[threadIdx.x] = inc - tot;
  }
  __syncthreads();
  if (threadIdx.x < 256) {
    unsigned wbase = 0;
    for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) wbase += sm.wsum[w];
    const unsigned d = threadIdx.x;
    sm.base[d] += wbase + hist[((size_t)blockIdx.y * 256 + d) * tiles + blockIdx.x] - sm.cnt[d * kSortWarps];
  }
  __syncthreads();
  for (int e = threadIdx.x; e < count; e += kSortThreads) {
    const u64 v = sm.v[e];
    dst[seg + (size_t)(sm.base[digit_of(v, shift)] + (unsigned)e)] = v;
  }
}

// ---- scores and statistics ------------------------------------------------------------------------------------------
// grid (ceil(n / 256), Dc).  Rank r + 1 of the pair at sorted position r: its Blom score to out[(s * 2C + k) * ld + dl]
// (skipped when out is null); with stats, the original draws at the positions of sp and the column's NaN flag.
__global__ void __launch_bounds__(256) k_rank_scores(long long n, int h, int C, int D, int d0, const float* __restrict__ hist,
                                                     const u64* __restrict__ pairs, float* __restrict__ out, int ld,
                                                     float* __restrict__ stats, StatPos sp) {
  const long long r = (long long)blockIdx.x * 256 + threadIdx.x;
  if (r >= n) return;
  const int dl = blockIdx.y;
  const u64 v = pairs[(size_t)dl * n + r];
  const unsigned j = (unsigned)v;
  const int k = (int)(j / (unsigned)h), s = (int)(j - (unsigned)k * (unsigned)h);
  if (out) {
    const double p = ((double)(r + 1) - 0.375) / ((double)n + 0.25);
    out[((size_t)s * (2 * C) + k) * ld + dl] = (float)normcdfinv(p);
  }
  if (!stats) return;
  float* st = stats + (size_t)dl * kStats;
#pragma unroll
  for (int q = 0; q < 6; ++q)
    if (r == sp.pos[q]) st[q] = hist[((size_t)(s + (k >= C ? h : 0)) * C + k % C) * D + d0 + dl];
  if (r == n - 1) st[6] = (unsigned)(v >> 32) == kNanKey ? 1.0f : 0.0f;
}

// out[(s * 2C + k) * Dc + dl] = upper ? x >= q_hi : x <= q_lo, compared in float64
__global__ void k_rank_indicator(int h, int C, int D, int d0, int Dc, const float* __restrict__ hist,
                                 const float* __restrict__ stats, StatPos sp, int upper, float* __restrict__ out) {
  const long long total = (long long)h * 2 * C * Dc;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int dl = (int)(e % Dc);
    const long long sk = e / Dc;
    const int k = (int)(sk % (2 * C)), s = (int)(sk / (2 * C));
    const float* st = stats + (size_t)dl * kStats;
    const double x = hist[((size_t)(s + (k >= C ? h : 0)) * C + k % C) * D + d0 + dl];
    const bool ind = upper ? x >= lerp_quantile(st[4], st[5], sp.t_hi) : x <= lerp_quantile(st[2], st[3], sp.t_lo);
    out[e] = ind ? 1.0f : 0.0f;
  }
}

__device__ __forceinline__ float nan_max(float a, float b) { return (a != a || b != b) ? __int_as_float(0x7fc00000) : fmaxf(a, b); }
__device__ __forceinline__ float nan_min(float a, float b) { return (a != a || b != b) ? __int_as_float(0x7fc00000) : fminf(a, b); }

// tmp = (R̂ bulk, R̂ fold, ESS lower, ESS upper) [4][Dc]; outputs at d0, each optional; a NaN column reports NaN
__global__ void k_rank_finish(int Dc, const float* __restrict__ stats, const float* __restrict__ tmp, float* rhat,
                              float* ess_bulk, float* ess_tail) {
  const int dl = blockIdx.x * blockDim.x + threadIdx.x;
  if (dl >= Dc) return;
  const bool nan = stats[(size_t)dl * kStats + 6] != 0.0f;
  const float qnan = __int_as_float(0x7fc00000);
  if (rhat) rhat[dl] = nan ? qnan : nan_max(tmp[dl], tmp[Dc + dl]);
  if (ess_bulk && nan) ess_bulk[dl] = qnan;
  if (ess_tail) ess_tail[dl] = nan ? qnan : nan_min(tmp[2 * Dc + dl], tmp[3 * Dc + dl]);
}

// ---- host --------------------------------------------------------------------------------------------------------------
inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// Scratch of one pass over Dc dimensions.  The second pair buffer doubles as the [h, 2C, Dc] score buffer once a sort
// has ended in the first; the tile histogram and the R̂ / ESS scratch are live at different times and share one region.
struct Layout {
  size_t pairs, hist_off, total_off, region, stats, tmp, bytes;
};
Layout layout(long long n, int h, int C, int Dc) {
  Layout L;
  L.pairs = align256(sizeof(u64) * (size_t)n * Dc);
  const long long tiles = n > kTile ? (n + kTile - 1) / kTile : 0;
  const size_t hist = align256(sizeof(unsigned) * 256 * (size_t)tiles * Dc);
  const size_t total = tiles ? align256(sizeof(unsigned) * 256 * (size_t)Dc) : 0;
  const size_t rhat = sizeof(float) * (2 * (size_t)(2 * C) * Dc + 4 + 4 * (size_t)Dc);
  const size_t ess = sizeof(float) * ess_scratch_floats(h, 2 * C, Dc);
  size_t region = hist + total;
  region = region > rhat ? region : rhat;
  region = region > ess ? region : ess;
  L.hist_off = 0;
  L.total_off = hist;
  L.region = align256(region);
  L.stats = align256(sizeof(float) * kStats * (size_t)Dc);
  L.tmp = align256(sizeof(float) * 4 * (size_t)Dc);
  L.bytes = 2 * L.pairs + L.region + L.stats + L.tmp;
  return L;
}

struct Bufs {
  u64 *a, *b;
  unsigned *hist, *total;
  float *region, *stats, *tmp;
};
Bufs carve(void* scratch, const Layout& L) {
  unsigned char* p = static_cast<unsigned char*>(scratch);
  Bufs B;
  B.a = reinterpret_cast<u64*>(p);
  B.b = reinterpret_cast<u64*>(p + L.pairs);
  unsigned char* r = p + 2 * L.pairs;
  B.hist = reinterpret_cast<unsigned*>(r + L.hist_off);
  B.total = reinterpret_cast<unsigned*>(r + L.total_off);
  B.region = reinterpret_cast<float*>(r);
  B.stats = reinterpret_cast<float*>(r + L.region);
  B.tmp = reinterpret_cast<float*>(r + L.region + L.stats);
  return B;
}

// The largest Dc <= D whose pass fits budget, rounded down to a multiple of 32 when that leaves at least 32 (so that
// k_ess_autocov's lanes stay full); 0 when one dimension does not fit.
int dims_per_pass(long long n, int h, int C, int D, size_t budget) {
  int lo = 0, hi = D;
  while (lo < hi) {
    const int mid = lo + (hi - lo + 1) / 2;
    if (layout(n, h, C, mid).bytes <= budget) lo = mid;
    else hi = mid - 1;
  }
  if (lo >= 32 && lo < D) lo -= lo % 32;
  return lo;
}

StatPos stat_positions(long long n, double prob) {
  StatPos sp;
  sp.pos[0] = (n - 1) / 2;
  sp.pos[1] = n / 2;  // ceil((n - 1) / 2)
  const double q[2] = {(1.0 - prob) / 2.0, (1.0 + prob) / 2.0};
  double t[2];
  for (int i = 0; i < 2; ++i) {
    const double v = q[i] * (double)(n - 1);
    const double fl = floor(v);
    long long lo = (long long)fl;
    lo = lo < 0 ? 0 : (lo > n - 1 ? n - 1 : lo);
    sp.pos[2 + 2 * i] = lo;
    sp.pos[3 + 2 * i] = lo + 1 < n ? lo + 1 : n - 1;
    t[i] = v - fl;
  }
  sp.t_lo = t[0];
  sp.t_hi = t[1];
  return sp;
}

// Segmented stable sort of Dc segments of n pairs; the result ends in B.a.
void sort_segments(const Bufs& B, long long n, int Dc, cudaStream_t s) {
  const int smem = (int)sizeof(SortSmem);
  if (n <= kTile) {
    cudaFuncSetAttribute(k_rank_sort_tile, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    k_rank_sort_tile<<<Dc, kSortThreads, smem, s>>>((int)n, B.a);
    return;
  }
  cudaFuncSetAttribute(k_rank_scatter, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  const int tiles = (int)((n + kTile - 1) / kTile);
  u64 *src = B.a, *dst = B.b;
  for (int shift = 0; shift < 32; shift += 8) {
    k_rank_hist<<<dim3(tiles, Dc), kSortThreads, 0, s>>>(n, tiles, shift, src, B.hist);
    k_rank_scan<<<dim3(256, Dc), 256, 0, s>>>(tiles, B.hist, B.total);
    k_rank_scatter<<<dim3(tiles, Dc), kSortThreads, smem, s>>>(n, tiles, shift, src, B.hist, B.total, dst);
    u64* t = src;
    src = dst;
    dst = t;
  }
}

struct Shape {
  int T, h, C, D;
  long long n;
};

// keys (bulk, or folded about the medians in B.stats) of dims [d0, d0 + Dc), sorted into B.a
void rank_chunk(const Shape& S, const float* history, int d0, int Dc, bool folded, const Bufs& B, cudaStream_t s) {
  const dim3 grid((unsigned)(2 * S.C * ((S.h + 31) / 32)), (unsigned)((Dc + 31) / 32));
  k_rank_keys<<<grid, dim3(32, 8), 0, s>>>(S.h, S.C, S.D, d0, Dc, S.n, history, folded ? B.stats : nullptr, B.a);
  sort_segments(B, S.n, Dc, s);
}
void score_chunk(const Shape& S, const float* history, int d0, int Dc, const Bufs& B, float* out, int ld, bool stats,
                 const StatPos& sp, cudaStream_t s) {
  const dim3 grid((unsigned)((S.n + 255) / 256), (unsigned)Dc);
  k_rank_scores<<<grid, 256, 0, s>>>(S.n, S.h, S.C, S.D, d0, history, B.a, out, ld, stats ? B.stats : nullptr, sp);
}

// shared argument checks: the shape and the pass width the scratch allows (or the rejection)
int rank_setup(bjx_handle_t h, const float* history, int32_t num_samples, void* scratch, size_t scratch_bytes, Shape& S,
               Layout& L, int& Dc) {
  if (!h || !history || !scratch) return bjx_fail(h, BJX_E_INVALID, "null argument");
  if (num_samples < 4) return bjx_fail(h, BJX_E_INVALID, "rank-normalised diagnostics need num_samples >= 4");
  S.T = num_samples;
  S.h = num_samples / 2;
  S.C = h->cfg.n_chains;
  S.D = h->cfg.dim;
  S.n = 2LL * S.C * S.h;
  if (S.n >= (1LL << 31))
    return bjx_fail(h, BJX_E_INVALID, "rank-normalised diagnostics need n = 2 * n_chains * (num_samples / 2) < 2^31 "
                                      "pooled draws per dimension");
  if ((reinterpret_cast<uintptr_t>(scratch) & 255u) != 0)
    return bjx_fail(h, BJX_E_INVALID, "scratch must be 256-byte aligned");
  Dc = dims_per_pass(S.n, S.h, S.C, S.D, scratch_bytes);
  if (Dc < 1)
    return bjx_fail(h, BJX_E_INVALID, "scratch too small: one dimension per pass needs " +
                                          std::to_string(layout(S.n, S.h, S.C, 1).bytes) + " bytes");
  L = layout(S.n, S.h, S.C, Dc);
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  return 0;
}

}  // namespace

extern "C" int64_t bjx_rank_diagnostics_scratch_bytes(int32_t num_samples, int32_t n_chains, int32_t dim,
                                                      int32_t dims_per_pass) {
  if (num_samples < 4 || n_chains < 1 || dim < 1 || dims_per_pass < 1) return -1;
  const int h = num_samples / 2;
  const int Dc = dims_per_pass < dim ? dims_per_pass : dim;
  return (int64_t)layout(2LL * n_chains * h, h, n_chains, Dc).bytes;
}

extern "C" int bjx_rank_normalize(bjx_handle_t h, const float* history, int32_t num_samples, int32_t folded, float* out,
                                  void* scratch, size_t scratch_bytes) {
  Shape S;
  Layout L;
  int Dc = 0;
  if (!out) return bjx_fail(h, BJX_E_INVALID, "null argument");
  int rc = rank_setup(h, history, num_samples, scratch, scratch_bytes, S, L, Dc);
  if (rc) return rc;
  const Bufs B = carve(scratch, L);
  const StatPos sp = stat_positions(S.n, 0.5);
  for (int d0 = 0; d0 < S.D; d0 += Dc) {
    const int dc = S.D - d0 < Dc ? S.D - d0 : Dc;
    rank_chunk(S, history, d0, dc, false, B, h->stream);
    score_chunk(S, history, d0, dc, B, folded ? nullptr : out + d0, S.D, folded != 0, sp, h->stream);
    if (folded) {
      rank_chunk(S, history, d0, dc, true, B, h->stream);
      score_chunk(S, history, d0, dc, B, out + d0, S.D, false, sp, h->stream);
    }
  }
  BJX_CHECK_LAUNCH("k_rank_normalize");
  return 0;
}

extern "C" int bjx_rank_diagnostics(bjx_handle_t h, const float* history, int32_t num_samples, double prob,
                                    float* rhat_out, float* ess_bulk_out, float* ess_tail_out, void* scratch,
                                    size_t scratch_bytes) {
  Shape S;
  Layout L;
  int Dc = 0;
  if (!(prob > 0.0 && prob < 1.0)) return bjx_fail(h, BJX_E_INVALID, "prob must be finite and in (0, 1)");
  int rc = rank_setup(h, history, num_samples, scratch, scratch_bytes, S, L, Dc);
  if (rc) return rc;
  const Bufs B = carve(scratch, L);
  const StatPos sp = stat_positions(S.n, prob);
  float* scores = reinterpret_cast<float*>(B.b);  // [h, 2C, dc], free once a sort has ended in B.a
  const cudaStream_t st = h->stream;
  for (int d0 = 0; d0 < S.D; d0 += Dc) {
    const int dc = S.D - d0 < Dc ? S.D - d0 : Dc;
    rank_chunk(S, history, d0, dc, false, B, st);
    score_chunk(S, history, d0, dc, B, (rhat_out || ess_bulk_out) ? scores : nullptr, dc, true, sp, st);
    if (ess_bulk_out) launch_ess(S.h, 2 * S.C, dc, scores, ess_bulk_out + d0, B.region, st);
    if (rhat_out) launch_rhat(S.h, 2 * S.C, dc, scores, B.tmp, B.region, st);
    if (ess_tail_out) {
      const unsigned blocks = (unsigned)((S.n * dc + 255) / 256 < 8 * 1024 ? (S.n * dc + 255) / 256 : 8 * 1024);
      for (int upper = 0; upper < 2; ++upper) {
        k_rank_indicator<<<blocks, 256, 0, st>>>(S.h, S.C, S.D, d0, dc, history, B.stats, sp, upper, scores);
        launch_ess(S.h, 2 * S.C, dc, scores, B.tmp + (2 + upper) * dc, B.region, st);
      }
    }
    if (rhat_out) {
      rank_chunk(S, history, d0, dc, true, B, st);
      score_chunk(S, history, d0, dc, B, scores, dc, false, sp, st);
      launch_rhat(S.h, 2 * S.C, dc, scores, B.tmp + dc, B.region, st);
    }
    k_rank_finish<<<(dc + 127) / 128, 128, 0, st>>>(dc, B.stats, B.tmp, rhat_out ? rhat_out + d0 : nullptr,
                                                    ess_bulk_out ? ess_bulk_out + d0 : nullptr,
                                                    ess_tail_out ? ess_tail_out + d0 : nullptr);
  }
  BJX_CHECK_LAUNCH("k_rank_diagnostics");
  return 0;
}
