// Batched dense linear map for the large-D dense metric / dense Gaussian target (SURVEY K8):
//   Y[R, N] = epilogue( X[R, K] . A[N, K]^T , Cin[R, N] )            (A symmetric: M^-1, precision; or L^-T)
// = the reference's `linear_map(M^-1, p)` / `-P x` / `L^-T z` (blackjax/util.py:23-61, lax.dot with
// precision="highest"; call sites mcmc/integrators.py:242, mcmc/metrics.py:263-270) for all chains at once.
//
// Hand-written sm_90a kernel: persistent CTAs, one producer warp issuing TMA (cp.async.bulk.tensor) operand loads into
// 128B-swizzled shared memory, two consumer warpgroups issuing wgmma.mma_async on them (each owns 64 rows of a 128 x 128
// output tile, float32 accumulators in registers), a STAGES-deep mbarrier ring between them.  A consumer keeps a second
// accumulator set: when a tile's K loop ends its sums move there, and its epilogue runs in slices under the next tile's
// MMAs, one slice after each of the first K blocks is issued.
//
// float32 accuracy on the fp16 tensor-core path.  One TF32/BF16/FP16 MMA (11/8/11-bit significands) cannot meet the
// 1e-5 parity tolerance, so every float32 operand is split into two binary16 terms x = x1 + x2 (+ a residual below
// 2^-22 |x|) and the three cross products above that residual are accumulated in float32:
//     x.a  ~=  x1 a1 + x2 a1 + x1 a2                      (dropped: x2 a2 and the residuals, each <= 2^-22 |x a|)
// Operand planes are stored [rows, 2, KP] = (x1 | x2): per 64-deep K block the producer stages FOUR tiles
// (x1, x2, a1, a2) and the consumers run the THREE products on them -- 2/3 of the shared-memory fill and L2 traffic of
// a plain K' = 3K GEMM over (x1|x2|x1).(a1|a1|a2), and 2/3 of the plane bytes in HBM.  What limits accuracy is then the
// tensor core's float32 accumulation, whose error grows about linearly with K: measured within 1e-5 of the row maximum
// up to K = 1028, 2.5e-5 at K = 4100 and 1e-4 at K = 18432 on random-sign data (DESIGN.md §3 "Accuracy").
// binary16 has a 5-bit exponent, so rows / matrices are lifted by a power of two before the split; the per-row
// epilogue factor alpha_r = coef_r * 2^-s_r * 2^-s_A undoes both exactly (and carries per-chain step sizes).
//
// Fused epilogue, straight from the accumulator registers:
//   lincomb      : y = alpha_r * acc + beta * Cin                 (q <- q + eps_c (p M^-1); v = M^-1 p; g = -(q P))
//   double kick  : y = alpha_r * acc + (alpha_r * acc + Cin)      (two half kicks between leapfrog steps,
//                                                                  integrators.py:134-141,235-239; two rounded FMAs)
//   planes       : the (x1 | x2) planes of y for the NEXT product, lifted by 2^s_r chosen from the row maximum the
//                  previous production of the same variable recorded (any lift that lands the true row maximum in
//                  [2^-3, 2^15.5) is exact to 2^-22 of the row maximum, an 18-binade window; rows that leave it are
//                  re-split by k_planes_fixup in bjx_dense.cu), plus this production's row maximum (atomic max).
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <mutex>

#include "bjx_gemm.h"

namespace bjx {
namespace {

constexpr int kBM = 128;                 // rows of X per tile (64 per consumer warpgroup)
constexpr int kBN = 128;                 // output columns per tile
constexpr int kBK = 64;                  // K per stage: one 128-byte swizzle row of binary16 per tile row
constexpr int kStages = 3;
constexpr int kThreads = 384;            // warpgroup 0: producer; warpgroups 1-2: consumers
constexpr int kTileBytes = kBM * kBK * 2;                  // one [128 x 64] binary16 tile (kBN == kBM)
constexpr int kStageBytes = 4 * kTileBytes;                // x1, x2, a1, a2
constexpr int kOffBar = kStages * kStageBytes;
// epilogue staging: per consumer warp 8 rows x 128 float32 of Y, rows padded by 4 floats against bank conflicts
constexpr int kStgLd = kBN + 4;
constexpr int kOffStg = kOffBar + 64;                      // after the 2 x kStages barriers, 16-byte aligned
constexpr int kSmemBytes = kOffStg + 8 * 8 * kStgLd * 4 + 1024;  // + slack to align the base to 1024
// A tile's epilogue runs in kSlices slices under the next tile's first kSlices K blocks (§3 of DESIGN.md: at D = 1024
// one slice under each K block measured faster than 8 slices)
constexpr int kSlices = 16;
constexpr int kHalfSlices = kSlices / 2;  // per half of the accumulator fragment (8 rows of each consumer warp)
static_assert(kSlices >= 2 && kSlices % 2 == 0 && kSlices <= 16, "whole halves, at most one staged row per slice");
static_assert(kBN == kBM, "the operand tiles of X and A share one size");
static_assert(kSmemBytes <= 232448, "over the 227 KB dynamic shared memory limit");

// ---- PTX wrappers -------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
  } while (!done);
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// operand tile [64 x 1 x 128] of a [K, 2, rows] plane tensor into shared memory, completion counted on `bar`
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// wgmma shared-memory matrix descriptor of a K-major [rows x 64] binary16 tile in the 128-byte swizzle TMA writes it
// in: 8-row groups 1024 bytes apart (stride byte offset), layout type SWIZZLE_128B (1).  Tiles start 1024-aligned.
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t smem_addr) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// wait until at most N committed wgmma groups of this warp are still in flight
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// the accumulators are written asynchronously: keep the compiler from reading them before the wait that completes them
__device__ __forceinline__ void fence_operands(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// per-thread register budget of the calling warpgroup (the CTA's total stays within 384 x 168)
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// d[64 x 128] += A[64 x 16] . B[128 x 16]^T, both operands K-major in shared memory, float32 accumulators in registers
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t desc_a, uint64_t desc_b) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, 1, 1, 1, 0, 0;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b)
      : "memory");
}

__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}
__device__ __forceinline__ float2 unpack_h2(uint32_t u) { return __half22float2(*reinterpret_cast<const __half2*>(&u)); }

}  // namespace

// ---- the kernel ---------------------------------------------------------------------------------------------
// Tiles t = (t / tiles_n, t % tiles_n) are dealt round-robin over the persistent CTAs; CTAs running side by side share
// one row block of X (the constant matrix stays L2-resident).
//   warp 0, lane 0   TMA producer: four tiles per stage into the ring
//   warpgroups 1-2   consumers: warpgroup w owns rows [64 (w-1), +64) of the tile; per stage 3 x 4 wgmma, and once
//                    they are issued the previous stage's group is waited for and that stage released (one arrival per
//                    consumer warp).  Then one slice of the PREVIOUS tile's epilogue runs from its saved accumulators
//                    while this block's group is in flight: a half's rows of Y staged in shared memory beside the ring,
//                    one staged row stored (Y and its two planes), or a half's row maxima recorded.  The epilogue's
//                    global inputs are loaded during the K loop of its own tile, and the CTA's last tile runs its
//                    epilogue whole after the loop.  The producer warpgroup runs on 40 registers per thread so that
//                    the consumers can hold both accumulator sets and those inputs (232).
// Slices and loads may run in any order relative to the tiles in flight: Y may alias Cin, but only elementwise (element
// (r, c) is read as Cin and written as Y by the same thread, and no two tiles share an element), the planes a launch
// writes are never the planes it reads (the momentum and position planes alternate between products), and the per-row
// arrays read (step sizes, unscales, stale maxima) are never among the same launch's outputs.
// Accumulator fragment of m64n128 (per warp of the warpgroup): d[4j + 2h + e] is row 16 warp + 8h + lane / 4,
// column 8j + 2 (lane % 4) + e.
__global__ void __launch_bounds__(kThreads, 1)
k_gemm_f16x3(const __grid_constant__ CUtensorMap tm_x,   // [K, 2, M]  binary16 planes of the activations
             const __grid_constant__ CUtensorMap tm_a,   // [K, 2, N]  binary16 planes of the constant matrix
             float* Y, const float* Cin, uint16_t* planes_out, const GemmEpilogue E, const int M, const int N, const int K,
             const int KP_out, const int tiles_n, const int n_tiles) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar0 = base + kOffBar;
  auto full_bar = [&](int s) { return bar0 + 8u * s; };
  auto empty_bar = [&](int s) { return bar0 + 8u * (kStages + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nkb = (K + kBK - 1) / kBK;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tm_x);
    prefetch_tmap(&tm_a);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full_bar(s), 1);    // the producer's arrive (+ the bytes of the four tiles)
      mbar_init(empty_bar(s), 8);   // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // Programmatic dependent launch: everything above may run while the previous kernel of the stream drains; nothing
  // below touches its outputs earlier.
  asm volatile("griddepcontrol.wait;" ::: "memory");

  if (warp < 4) {
    // ===== TMA producer.  The whole warpgroup hands its registers to the consumers (which hold the accumulators and
    // the prefetched epilogue inputs) before warps 1-3 leave.
    setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      int s = 0;
      uint32_t ph = 0;
      for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const int m0 = (t / tiles_n) * kBM, n0 = (t % tiles_n) * kBN;
        for (int kb = 0; kb < nkb; ++kb) {
          mbar_wait(empty_bar(s), ph ^ 1u);
          mbar_expect_tx(full_bar(s), (uint32_t)kStageBytes);
          const uint32_t st = base + (uint32_t)s * kStageBytes;
          tma_load_3d(st, &tm_x, full_bar(s), kb * kBK, 0, m0);
          tma_load_3d(st + kTileBytes, &tm_x, full_bar(s), kb * kBK, 1, m0);
          tma_load_3d(st + 2 * kTileBytes, &tm_a, full_bar(s), kb * kBK, 0, n0);
          tma_load_3d(st + 3 * kTileBytes, &tm_a, full_bar(s), kb * kBK, 1, n0);
          if (++s == kStages) { s = 0; ph ^= 1u; }
        }
      }
    }
    return;
  }

  // ===== consumers
  setmaxnreg_inc<232>();
  const int wg = (warp >> 2) - 1, wq = warp & 3;
  const float mat_unscale = E.mat_unscale ? E.mat_unscale[0] : 1.0f;
  float* stg = reinterpret_cast<float*>(smem_raw + (base - smem_u32(smem_raw)) + kOffStg) + (warp - 4) * 8 * kStgLd;

  // One K block of the current tile: its MMAs are issued (k_issue) before the wait for block kb - 1's, whose stage is
  // released only then (k_retire), so one wgmma group stays in flight.  wgmmas on one accumulator complete in issue
  // order, so the sums are those of a serial loop.
  float acc[64];
  int s = 0, s_prev = 0;
  uint32_t ph = 0;
  auto k_issue = [&]() {
    mbar_wait(full_bar(s), ph);
    const uint32_t st = base + (uint32_t)s * kStageBytes;
    const uint32_t xo = (uint32_t)wg * (64u * kBK * 2u);  // this warpgroup's 64 rows of the X tiles
    const uint64_t dx1 = wgmma_desc(st + xo), dx2 = wgmma_desc(st + kTileBytes + xo);
    const uint64_t da1 = wgmma_desc(st + 2 * kTileBytes), da2 = wgmma_desc(st + 3 * kTileBytes);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kBK / 16; ++k) wgmma_m64n128k16(acc, dx1 + 2u * k, da1 + 2u * k);  // +32 bytes per K step
#pragma unroll
    for (int k = 0; k < kBK / 16; ++k) wgmma_m64n128k16(acc, dx2 + 2u * k, da1 + 2u * k);
#pragma unroll
    for (int k = 0; k < kBK / 16; ++k) wgmma_m64n128k16(acc, dx1 + 2u * k, da2 + 2u * k);
    wgmma_commit();
  };
  auto k_retire = [&](const int kb) {
    wgmma_wait<1>();
    if (kb > 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar(s_prev));
    }
    s_prev = s;
    if (++s == kStages) { s = 0; ph ^= 1u; }
  };

  // The global inputs of the current tile's epilogue, loaded while its MMAs run: per row of the thread's two the step
  // size, the activations' unscale and the stale maximum that chooses the lift (combined only once the tile's K loop
  // is done, so that no instruction inside it waits for them), and the thread's 32 float2 of Cin.
  float in_alpha[2], in_unscale[2], in_max[2];
  float2 cin[2][kBN / 8];
  auto load_inputs = [&](const int m0, const int n0) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = m0 + 64 * wg + 16 * wq + 8 * h + (lane >> 2);
      in_alpha[h] = 1.0f;
      in_unscale[h] = 1.0f;
      in_max[h] = 0.0f;
      if (r < M) {
        if (E.alpha_dev) in_alpha[h] = E.alpha_dev[r];
        if (E.x_unscale) in_unscale[h] = E.x_unscale[r];
        if (E.planes) in_max[h] = E.stale_max[r];
      }
#pragma unroll
      for (int j = 0; j < kBN / 8; ++j) {
        const int c = n0 + 8 * j + 2 * (lane & 3);
        cin[h][j] = make_float2(0.f, 0.f);
        if (E.has_cin && r < M && c < N) cin[h][j] = *reinterpret_cast<const float2*>(Cin + (size_t)r * N + c);
      }
    }
  };

  // The finished tile whose epilogue is still to run: its accumulators, per-row epilogue factors and lifts, and origin.
  float prev[64], pal[2] = {0.f, 0.f}, psc[2] = {1.f, 1.f};
  int pm0 = 0, pn0 = 0;
  bool pending = false;
  float amax = 0.f;  // this thread's part of the current half's row maximum, from its staging to its atomicMax

  // Slice e of that epilogue (two rows per thread, two adjacent columns per fragment register pair).  Y goes through
  // this warp's staging rows in shared memory, so that every global store of the warp writes whole rows (a fragment
  // store would touch 8 rows with 32 bytes each); the planes of Y are split from the staged rows, four columns per lane.
  // Half h = e / kHalfSlices of the fragment is staged by its first slice, its 8 staged rows are stored over its
  // kHalfSlices slices, and its last slice records the row maxima.
  auto epilogue_slice = [&](const int e) {
    const int h = e / kHalfSlices, j = e % kHalfSlices;
    const int r0 = pm0 + 64 * wg + 16 * wq + 8 * h;  // the warp's 8 rows of this half
    const int r = r0 + (lane >> 2);
    const bool live = r < M;
    if (j == 0) {
      const float al = pal[h];
      amax = 0.f;
#pragma unroll
      for (int jj = 0; jj < kBN / 8; ++jj) {
        const int c = pn0 + 8 * jj + 2 * (lane & 3);
        if (!live || c >= N) continue;
        const float a0 = prev[4 * jj + 2 * h], a1 = prev[4 * jj + 2 * h + 1];
        float2 y;
        if (E.has_cin) {
          const float2 cv = cin[h][jj];
          if (E.double_kick) {
            y.x = fmaf(al, a0, fmaf(al, a0, cv.x));
            y.y = fmaf(al, a1, fmaf(al, a1, cv.y));
          } else {
            y.x = fmaf(al, a0, E.beta * cv.x);
            y.y = fmaf(al, a1, E.beta * cv.y);
          }
        } else {
          y = make_float2(al * a0, al * a1);
        }
        *reinterpret_cast<float2*>(stg + (lane >> 2) * kStgLd + (c - pn0)) = y;
        if (E.planes) amax = fmaxf(amax, fmaxf(fabsf(y.x), fabsf(y.y)));
      }
      __syncwarp();
    }
    const int cw = pn0 + 4 * lane;  // the four columns this lane stores of every staged row
#pragma unroll
    for (int i = 8 * j / kHalfSlices; i < 8 * (j + 1) / kHalfSlices; ++i) {
      const float sci = __shfl_sync(0xffffffffu, psc[h], 4 * i);
      if (r0 + i >= M || cw >= N) continue;
      const float4 y = *reinterpret_cast<const float4*>(stg + i * kStgLd + 4 * lane);
      *reinterpret_cast<float4*>(Y + (size_t)(r0 + i) * N + cw) = y;
      if (E.planes) {
        const float s0 = y.x * sci, s1 = y.y * sci, s2 = y.z * sci, s3 = y.w * sci;
        const uint32_t h01 = pack_h2(s0, s1), h23 = pack_h2(s2, s3);
        const float2 f01 = unpack_h2(h01), f23 = unpack_h2(h23);
        uint16_t* pri = planes_out + (size_t)(r0 + i) * 2 * KP_out + cw;
        *reinterpret_cast<uint2*>(pri) = make_uint2(h01, h23);
        *reinterpret_cast<uint2*>(pri + KP_out) =
            make_uint2(pack_h2(s0 - f01.x, s1 - f01.y), pack_h2(s2 - f23.x, s3 - f23.y));
      }
    }
    if (j == kHalfSlices - 1) {
      __syncwarp();  // the staging rows are rewritten by the next half
      if (E.planes) {  // the four lanes of a row hold its 128 columns of this tile
        amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
        amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
        if (live && (lane & 3) == 0) {
          atomicMax(reinterpret_cast<int*>(E.next_max) + r, __float_as_int(amax));
          E.zero_max[r] = 0.f;
          if (pn0 == 0) E.out_unscale[r] = 1.0f / psc[h];  // the tile of the first column block writes the lift
        }
      }
    }
  };

  for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    const int m0 = (t / tiles_n) * kBM, n0 = (t % tiles_n) * kBN;
    if (!pending) load_inputs(m0, n0);
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    // The previous tile's epilogue runs under this tile's first kSlices K blocks, one slice behind each block's issue.
    // Its Cin registers are free once its second half is staged, and this tile's inputs are loaded into them then.
#pragma unroll
    for (int e = 0; e < kSlices; ++e) {
      if (e < nkb) k_issue();
      if (e < nkb) k_retire(e);
      if (pending) {
        epilogue_slice(e);
        if (e == kHalfSlices) load_inputs(m0, n0);
      }
    }
    for (int kb = kSlices; kb < nkb; ++kb) {
      k_issue();
      k_retire(kb);
    }
    wgmma_wait<0>();
    fence_operands(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(empty_bar(s_prev));

    // hand the tile over to the next tile's K loop
#pragma unroll
    for (int i = 0; i < 64; ++i) prev[i] = acc[i];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = m0 + 64 * wg + 16 * wq + 8 * h + (lane >> 2);
      float al = E.alpha, sc = 1.0f;
      if (r < M) {
        if (E.alpha_dev) al = in_alpha[h] * E.alpha;
        al = al * in_unscale[h] * mat_unscale;
        if (E.planes) sc = plane_lift(in_max[h]);
      }
      pal[h] = al;
      psc[h] = sc;
    }
    pm0 = m0;
    pn0 = n0;
    pending = true;
  }
  // the last tile's epilogue, whole
  if (pending) {
#pragma unroll
    for (int e = 0; e < kSlices; ++e) epilogue_slice(e);
  }
}

namespace {
// ---- host side ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) == cudaSuccess &&
        qr == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

// planes tensor [rows, 2, KP] binary16 seen as (K, 2, rows): box (64, 1, 128), 128-byte swizzle; out-of-range rows
// and K columns are filled with zeros
bool make_plane_map(CUtensorMap* m, const void* ptr, int rows, int K, int KP) {
  const cuuint64_t dims[3] = {(cuuint64_t)K, 2, (cuuint64_t)rows};
  const cuuint64_t strides[2] = {(cuuint64_t)KP * 2, (cuuint64_t)KP * 4};
  const cuuint32_t box[3] = {(cuuint32_t)kBK, 1, (cuuint32_t)kBM};
  const cuuint32_t es[3] = {1, 1, 1};
  return encode_fn()(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(ptr), dims, strides, box, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

int max_ctas() {  // one CTA per SM (the ring takes most of the shared memory)
  static int cached = 0;
  static std::once_flag once;
  std::call_once(once, [] {
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaFuncSetAttribute(k_gemm_f16x3, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
    cached = sms > 0 ? sms : 1;
  });
  return cached;
}

}  // namespace

int gemm_f16x3(const GemmCall& g, cudaStream_t stream) {
  if (!encode_fn()) return 1;
  if (g.M <= 0 || g.N <= 0 || g.K <= 0 || (g.N & 3) || (g.KP & 7) || (g.KP_out & 7)) return 2;
  CUtensorMap tx, ta;
  if (!make_plane_map(&tx, g.x_planes, g.M, g.K, g.KP)) return 3;
  if (!make_plane_map(&ta, g.a_planes, g.N, g.K, g.KP)) return 4;
  const int tiles_m = (g.M + kBM - 1) / kBM, tiles_n = (g.N + kBN - 1) / kBN;
  const int n_tiles = tiles_m * tiles_n;
  const int ctas = n_tiles < max_ctas() ? n_tiles : max_ctas();
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(ctas);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = kSmemBytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;  // prologue overlaps the previous kernel's tail
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, k_gemm_f16x3, tx, ta, g.Y, g.epi.has_cin ? g.Cin : nullptr,
                                           g.epi.planes ? g.planes_out : nullptr, g.epi, g.M, g.N, g.K, g.KP_out, tiles_n,
                                           n_tiles);
  return e == cudaSuccess ? 0 : 8;
}

}  // namespace bjx
