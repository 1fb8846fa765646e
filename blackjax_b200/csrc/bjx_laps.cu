// LAPS, the ensemble MCLMC warm-up (blackjax/adaptation/laps.py, laps_burn_in.py, eca.py): initialisation, the unadjusted
// burn-in with its ensemble averages and early stop, the phase switch, and the adjusted phase with the bisection of the
// step size, all on the handle's stream.
//
// Keys of a phase key k (laps.py:190, eca.py:243-249): key_sampling, key_adaptation = split(k); chain c at step t uses
// split(key_sampling, (N, T))[c, t] = fold_in(key_sampling, c T + t), every chain the adaptation key
// split(key_adaptation, T)[t] = fold_in(key_adaptation, t).
//
// The ensemble averages are sums over chains divided by N.  Every sum has one order fixed by N alone: the per-CTA records of
// k_laps_burn_in / k_laps_rowstats are added in block order by two k_laps_colsum passes, and the single-CTA updates reduce
// over dimensions with a fixed tree.  No float atomics: two runs are bit-identical.  The records are raw sums, so that
// records gathered from several ranks can be summed the same way.
#include <math.h>

#include "../../include/bjx.h"
#include "bjx_internal.h"
#include "bjx_launch.cuh"
#include "bjx_handle.h"

using namespace bjx;

namespace {

constexpr int kZRows = 100;       // equipartition_fullrank's Hutchinson probes (laps_burn_in.py:217)
constexpr int kStatGrid = 512;    // CTAs of k_laps_rowstats
constexpr int kMergeGroup = 32;   // records per partial sum of the first k_laps_colsum pass
constexpr int kUpd = 1024;        // threads of the single-CTA updates

__host__ __device__ inline size_t up4(size_t n) { return (n + 3) & ~(size_t)3; }
inline int n_groups(int rows, int group) { return (rows + group - 1) / group; }
inline int stat_grid(int C) { return C < kStatGrid ? C : kStatGrid; }
inline int zgx_chunks(int C) { return std::max(1, std::min(64, C / 256)); }

// Offsets (floats) into the caller's state buffer.
struct Layout {
  int C, D, rows, equi;
  size_t imm, hist, m1, rec1, part1, z, a, bp, keys, eps, acc, rec2, part2, m2, total;
  Layout(int C_, int D_, int save_num, int equi_full) : C(C_), D(D_), rows(save_num), equi(equi_full) {
    const size_t W1 = 3 * (size_t)D + 4, W2 = (size_t)D + 1;
    const int G1 = laps_grid(C), G2 = stat_grid(C);
    imm = LS_HDR;
    hist = imm + up4(D);
    m1 = hist + up4((size_t)rows * D);
    rec1 = m1 + up4(W1);
    part1 = rec1 + up4((size_t)G1 * W1);
    z = part1 + up4((size_t)n_groups(G1, kMergeGroup) * W1);
    a = z + (equi ? up4((size_t)kZRows * D) : 0);
    bp = a + (equi ? up4((size_t)kZRows * C) : 0);
    keys = bp + (equi ? up4((size_t)zgx_chunks(C) * kZRows * D) : 0);
    eps = keys + up4(2 * (size_t)C);
    acc = eps + up4(C);
    rec2 = acc + up4(C);
    part2 = rec2 + up4((size_t)G2 * W2);
    m2 = part2 + up4((size_t)n_groups(G2, kMergeGroup) * W2);
    total = m2 + up4(W2);
  }
};

__device__ __forceinline__ int* ihdr(float* s) { return reinterpret_cast<int*>(s); }

// deterministic block reductions over kUpd threads
__device__ float block_sum(float v, float* red) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) red[threadIdx.x] = __fadd_rn(red[threadIdx.x], red[threadIdx.x + o]);
    __syncthreads();
  }
  const float r = red[0];
  __syncthreads();
  return r;
}
__device__ __forceinline__ float nan_max(float a, float b) { return (isnan(a) || a > b) ? a : b; }  // jnp.max
__device__ float block_max(float v, float* red) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) red[threadIdx.x] = nan_max(red[threadIdx.x], red[threadIdx.x + o]);
    __syncthreads();
  }
  const float r = red[0];
  __syncthreads();
  return r;
}

// out[g, col] = sum of in[r, col] over the rows r of group g, in row order.  A stopped state (if given) skips the pass.
__global__ void k_laps_colsum(int rows, int width, int group, const float* __restrict__ in, float* __restrict__ out,
                              const float* state) {
  if (state && laps_stopped(state)) return;
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= width) return;
  const int r0 = blockIdx.y * group, r1 = min(rows, r0 + group);
  float s = 0.f;
  for (int r = r0; r < r1; ++r) s = __fadd_rn(s, in[(size_t)r * width + col]);
  out[(size_t)blockIdx.y * width + col] = s;
}

void merge(int rows, int width, const float* rec, float* part, float* out, const float* state, cudaStream_t s) {
  const int g = n_groups(rows, kMergeGroup);
  k_laps_colsum<<<dim3(blocks_for(width, 256), g), 256, 0, s>>>(rows, width, kMergeGroup, rec, part, state);
  k_laps_colsum<<<dim3(blocks_for(width, 256), 1), 256, 0, s>>>(g, width, g, part, out, state);
}

// Per-CTA sums over a fixed range of chains: rec[b] = (sum -x g [D], sum acc) when with_x, else only the acceptance.
__global__ void k_laps_rowstats(int C, int D, const float* __restrict__ q, const float* __restrict__ g,
                                const float* __restrict__ acc, int with_x, float* __restrict__ rec) {
  const int cs = (C + gridDim.x - 1) / gridDim.x;
  const int c0 = blockIdx.x * cs, c1 = min(C, c0 + cs);
  float* r = rec + (size_t)blockIdx.x * (D + 1);
  if (with_x) {
    for (int d = threadIdx.x; d < D; d += blockDim.x) {
      float s = 0.f;
      for (int c = c0; c < c1; ++c) s = __fadd_rn(s, __fmul_rn(-q[(size_t)c * D + d], g[(size_t)c * D + d]));
      r[d] = s;
    }
  }
  if (threadIdx.x == 0) {
    float s = 0.f;
    if (acc)
      for (int c = c0; c < c1; ++c) s = __fadd_rn(s, acc[c]);
    r[D] = s;
  }
}

// velocity = g / |g| (_normalized_flatten_array, tolerance 1e-13), one warp per chain
__global__ void k_laps_velocity(int C, int D, const float* __restrict__ g, float* __restrict__ u) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (c >= C) return;
  const float* row = g + (size_t)c * D;
  float ss = 0.f;
  for (int e = lane; e < D; e += 32) ss = __fmaf_rn(row[e], row[e], ss);
  const float n = sqrtf(warp_sum(ss));
  for (int e = lane; e < D; e += 32) u[(size_t)c * D + e] = n > 1e-13f ? __fdiv_rn(row[e], n) : row[e];
}

// dimension i of every velocity times -2 (E_i < 1) + 1, E_i = mean over chains of -x_i g_i (laps_burn_in.py:147-158)
__global__ void k_laps_signs(int C, int D, const float* __restrict__ sums, float* __restrict__ u) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)C * D) return;
  const int d = (int)(i % D);
  if (__fdiv_rn(sums[d], (float)C) < 1.0f) u[i] = -u[i];
}

// The burn-in's initial adaptation state (laps_burn_in.py:256-272): L = inf, eps = 0.01 sqrt(D), M^-1 = 1, empty history.
__global__ void k_laps_state_init(int D, int rows, float* state) {
  for (int i = threadIdx.x; i < D; i += blockDim.x) state[LS_HDR + i] = 1.0f;
  float* hist = state + LS_HDR + up4(D);
  for (size_t i = threadIdx.x; i < (size_t)rows * D; i += blockDim.x) hist[i] = 0.f;
  if (threadIdx.x == 0) {
    state[LS_L] = __int_as_float(0x7f800000);
    state[LS_EPS] = __fmul_rn(0.01f, sqrtf((float)D));
    ihdr(state)[LS_COUNT] = 0;
    ihdr(state)[LS_STOP] = 0;
    state[LS_EEVPD] = 1e-3f;
    state[LS_EEVPD_W] = 1e-3f;
    state[LS_EQUI_FULL] = __int_as_float(0x7fc00000);
  }
}

// Z = rademacher(key_adaptation_t, (100, D)) = 2 (uniform < 0.5) - 1
__global__ void k_laps_rademacher(int D, uint32_t ka, uint32_t kb, float* __restrict__ z, const float* state) {
  if (laps_stopped(state)) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= kZRows * D) return;
  z[i] = uniform01(Key{ka, kb}, (uint32_t)i) < 0.5f ? 1.0f : -1.0f;
}

// a[k, c] = Z[k] . g_c, one warp per chain
__global__ void k_laps_zg(int C, int D, const float* __restrict__ z, const float* __restrict__ g, float* __restrict__ a,
                          const float* state) {
  if (laps_stopped(state)) return;
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (c >= C) return;
  const float* row = g + (size_t)c * D;
  for (int k = 0; k < kZRows; ++k) {
    float s = 0.f;
    for (int e = lane; e < D; e += 32) s = __fmaf_rn(z[(size_t)k * D + e], row[e], s);
    s = warp_sum(s);
    if (lane == 0) a[(size_t)k * C + c] = s;
  }
}

// bp[chunk, k, d] = sum over the chunk's chains c of a[k, c] x[c, d], chains in order; 128 dimensions per CTA
__global__ void __launch_bounds__(128) k_laps_zgx(int C, int D, const float* __restrict__ a, const float* __restrict__ x,
                                                  float* __restrict__ bp, const float* state) {
  if (laps_stopped(state)) return;
  __shared__ float as[kZRows][32];
  const int d = blockIdx.x * 128 + threadIdx.x;
  const int cs = (C + gridDim.y - 1) / gridDim.y;
  const int c0 = blockIdx.y * cs, c1 = min(C, c0 + cs);
  float acc[kZRows];
#pragma unroll
  for (int k = 0; k < kZRows; ++k) acc[k] = 0.f;
  for (int cb = c0; cb < c1; cb += 32) {
    const int n = min(32, c1 - cb);
    __syncthreads();
    for (int i = threadIdx.x; i < kZRows * 32; i += 128) {
      const int k = i / 32, j = i % 32;
      as[k][j] = j < n ? a[(size_t)k * C + cb + j] : 0.f;
    }
    __syncthreads();
    if (d < D) {
      for (int j = 0; j < n; ++j) {
        const float xv = x[(size_t)(cb + j) * D + d];
#pragma unroll
        for (int k = 0; k < kZRows; ++k) acc[k] = __fmaf_rn(as[k][j], xv, acc[k]);
      }
    }
  }
  if (d < D) {
#pragma unroll
    for (int k = 0; k < kZRows; ++k) bp[((size_t)blockIdx.y * kZRows + k) * D + d] = acc[k];
  }
}

// equi_full = mean((Z + B / N)^2) / D (equipartition_fullrank_loss, laps_burn_in.py:226-228) into LS_EQUI_FULL
__global__ void __launch_bounds__(kUpd) k_laps_equi_full(int C, int D, int chunks, const float* __restrict__ z,
                                                          const float* __restrict__ bp, float* state) {
  if (laps_stopped(state)) return;
  __shared__ float red[kUpd];
  const int n = kZRows * D;
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    float b = 0.f;
    for (int ch = 0; ch < chunks; ++ch) b = __fadd_rn(b, bp[(size_t)ch * n + i]);
    const float v = __fadd_rn(z[i], __fdiv_rn(b, (float)C));
    s = __fmaf_rn(v, v, s);
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) state[LS_EQUI_FULL] = __fdiv_rn(__fdiv_rn(s, (float)n), (float)D);
}

struct BurnInUpdate {
  int C, D, rows, bias_type, early_stop, t;
  float alpha, c, r_end;
};

// Adaptation.update (laps_burn_in.py:292-364) and the stop rule (:366-368, eca.py:119-156) from the merged sums m [3 D + 4].
// The history ring holds the ensemble means of x of the last `rows` steps; slot t % rows takes step t's, and the weighted
// averages of contract_history run over the filled slots newest first.  info (optional) receives
// (L, step_size, EEVPD_wanted, EEVPD, equi_diag, equi_full, r_max, r_avg, entropy) of the state before the update.
__global__ void __launch_bounds__(kUpd) k_laps_update(BurnInUpdate U, const float* __restrict__ m, float* state,
                                                       float* info) {
  if (laps_stopped(state)) return;
  __shared__ float red[kUpd];
  const int D = U.D;
  const float N = (float)U.C;
  float* imm = state + LS_HDR;
  float* hist = imm + up4(D);
  const int slot = U.t % U.rows, filled = min(U.t + 1, U.rows);
  float sv = 0.f, se = 0.f, sr = 0.f, mr = -__int_as_float(0x7f800000);
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    const float emg = __fdiv_rn(m[d], N), ex = __fdiv_rn(m[D + d], N), exsq = __fdiv_rn(m[2 * D + d], N);
    const float v = __fsub_rn(exsq, __fmul_rn(ex, ex));
    imm[d] = v;
    sv = __fadd_rn(sv, v);
    const float om = __fsub_rn(1.0f, emg);
    se = __fadd_rn(se, __fmul_rn(om, om));
    hist[(size_t)slot * D + d] = ex;
    float s1 = 0.f, s2 = 0.f;
    for (int j = 0; j < filled; ++j) {
      const float h = hist[(size_t)((slot - j + U.rows) % U.rows) * D + d];
      s1 = __fadd_rn(s1, h);
      s2 = __fadd_rn(s2, __fmul_rn(h, h));
    }
    const float a1 = __fdiv_rn(s1, (float)filled), a2 = __fdiv_rn(s2, (float)filled);
    const float sq = __fmul_rn(a1, a1);
    const float r = __fdiv_rn(__fsub_rn(a2, sq), sq);
    sr = __fadd_rn(sr, r);
    mr = nan_max(mr, r);
  }
  sv = block_sum(sv, red);
  se = block_sum(se, red);
  sr = block_sum(sr, red);
  mr = block_max(mr, red);
  if (threadIdx.x != 0) return;
  const float* s = m + 3 * D;
  const float E = __fdiv_rn(s[0], N), Esq = __fdiv_rn(s[1], N), nans = __fdiv_rn(s[2], N), ent = __fdiv_rn(s[3], N);
  const float L = __fmul_rn(__fmul_rn(U.alpha, sqrtf(__fdiv_rn(sv, (float)D))), sqrtf((float)D));
  const float eevpd = __fdiv_rn(__fsub_rn(Esq, __fmul_rn(E, E)), (float)D);
  const float equi_diag = __fdiv_rn(se, (float)D), r_avg = __fdiv_rn(sr, (float)D);
  const float equi_full = state[LS_EQUI_FULL];
  const float bias = U.bias_type == 0 ? mr : U.bias_type == 1 ? r_avg : U.bias_type == 2 ? equi_full : equi_diag;
  const float wanted = __fmul_rn(U.c, powf(bias, 0.375f));
  float f = powf(__fdiv_rn(wanted, eevpd), 1.0f / 6.0f);
  f = f < 0.3f ? 0.3f : (f > 3.0f ? 3.0f : f);  // jnp.clip, NaN stays NaN
  if (nans > 0.f) f = 0.5f;
  if (info) {
    float* row = info + (size_t)U.t * 9;
    row[0] = state[LS_L];
    row[1] = state[LS_EPS];
    row[2] = wanted;
    row[3] = eevpd;
    row[4] = equi_diag;
    row[5] = equi_full;
    row[6] = mr;
    row[7] = r_avg;
    row[8] = ent;
  }
  state[LS_L] = L;
  state[LS_EPS] = __fmul_rn(state[LS_EPS], f);
  state[LS_EEVPD] = eevpd;
  state[LS_EEVPD_W] = wanted;
  ihdr(state)[LS_COUNT] = U.t + 1;
  if (U.early_stop && !(mr > U.r_end) && U.t >= U.rows) ihdr(state)[LS_STOP] = 1;
}

// laps.py:250-257, 76: eps /= sqrt(mean(M^-1)) with diagonal preconditioning; bisection bounds [-inf, inf], not terminated
__global__ void __launch_bounds__(kUpd) k_laps_switch(int D, int diag, float* state) {
  __shared__ float red[kUpd];
  float s = 0.f;
  for (int d = threadIdx.x; d < D; d += blockDim.x) s = __fadd_rn(s, state[LS_HDR + d]);
  s = block_sum(s, red);
  if (threadIdx.x != 0) return;
  if (diag) state[LS_EPS] = __fdiv_rn(state[LS_EPS], sqrtf(__fdiv_rn(s, (float)D)));
  state[LS_LO] = -__int_as_float(0x7f800000);
  state[LS_HI] = __int_as_float(0x7f800000);
  state[LS_TERM] = 0.f;
}

// keys[c] = fold_in(key_sampling, (chain_offset + c) T + t)
__global__ void k_laps_keys(int C, uint32_t ka, uint32_t kb, uint32_t off, uint32_t T, uint32_t t, uint32_t* out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const Key k = fold_in(Key{ka, kb}, (off + (uint32_t)c) * T + t);
  out[2 * c] = k.a;
  out[2 * c + 1] = k.b;
}

// Adaptation.update of the adjusted phase (laps.py:90-120) with bisection_monotonic_fn (step_size.py:262-304) from the
// merged sums m [D + 1]; info (optional) receives (L = eps steps_per_sample, step_size, acc_prob, equi_diag).
__global__ void __launch_bounds__(kUpd) k_laps_bisect(int C, int D, int with_x, const float* __restrict__ m, float target,
                                                       int steps_per_sample, int t, float* state, float* info) {
  __shared__ float red[kUpd];
  const float N = (float)C;
  float se = 0.f;
  if (with_x)
    for (int d = threadIdx.x; d < D; d += blockDim.x) {
      const float om = __fsub_rn(1.0f, __fdiv_rn(m[d], N));
      se = __fadd_rn(se, __fmul_rn(om, om));
    }
  se = block_sum(se, red);
  if (threadIdx.x != 0) return;
  const float acc = __fdiv_rn(m[D], N);
  const float eps = state[LS_EPS];
  if (info) {
    float* row = info + (size_t)t * 4;
    row[0] = __fmul_rn(eps, (float)steps_per_sample);
    row[1] = eps;
    row[2] = acc;
    row[3] = with_x ? __fdiv_rn(se, (float)D) : __int_as_float(0x7fc00000);
  }
  const float shift = 0.6931471805599453f;  // log 2
  float lo = state[LS_LO], hi = state[LS_HI];
  const float x = logf(eps);
  float xn;
  if (acc > target) {
    lo = nan_max(lo, x);
    xn = __fadd_rn(lo, shift);
  } else {
    hi = (isnan(hi) || hi < x) ? hi : x;  // jnp.min
    if (isnan(x)) hi = x;
    xn = __fsub_rn(hi, shift);
  }
  if (isfinite(lo) && isfinite(hi)) xn = __fdiv_rn(__fadd_rn(lo, hi), 2.0f);
  const float term = state[LS_TERM];
  state[LS_EPS] = __fadd_rn(__fmul_rn(term, eps), __fmul_rn(__fsub_rn(1.0f, term), expf(xn)));
  state[LS_LO] = lo;
  state[LS_HI] = hi;
  state[LS_TERM] = (fabsf(__fsub_rn(acc, target)) < 0.03f || term != 0.f) ? 1.0f : 0.0f;
}

int laps_supported(bjx_handle_t h, int save_num) {
  int rc = mclmc_transition_supported(h, "LAPS");
  if (rc) return rc;
  if (h->metric_kind != BJX_METRIC_DIAG)
    return bjx_fail(h, BJX_E_UNSUPPORTED, "LAPS shares one diagonal metric [dim] between all chains");
  if (save_num < 1) return bjx_fail(h, BJX_E_INVALID, "LAPS needs save_num = rint(save_frac * num_steps1) >= 1");
  return 0;
}

}  // namespace

extern "C" int64_t bjx_laps_state_floats(int32_t n_chains, int32_t dim, int32_t save_num, int32_t equi_full) {
  if (n_chains < 1 || dim < 1 || save_num < 1) return -1;
  return (int64_t)Layout(n_chains, dim, save_num, equi_full ? 1 : 0).total;
}

extern "C" int bjx_laps_init(bjx_handle_t h, const float* q, float* logp, float* grad, float* u, float* state,
                             int32_t save_num) {
  const void* ptrs[] = {q, grad, u, state};
  int rc = check_ready(h, true, ptrs, 4);
  if (rc) return rc;
  if (!logp) return bjx_fail(h, BJX_E_INVALID, "null argument");
  if ((rc = laps_supported(h, save_num))) return rc;
  if ((rc = bjx_init_state(h, q, logp, grad))) return rc;
  const int C = h->cfg.n_chains, D = h->cfg.dim;
  const cudaStream_t s = h->stream;
  const Layout Lo(C, D, save_num, 0);
  k_laps_velocity<<<blocks_for(C, 8), 256, 0, s>>>(C, D, grad, u);
  k_laps_rowstats<<<stat_grid(C), 256, 0, s>>>(C, D, q, grad, nullptr, 1, state + Lo.rec2);
  merge(stat_grid(C), D + 1, state + Lo.rec2, state + Lo.part2, state + Lo.m2, nullptr, s);
  k_laps_signs<<<blocks_for((long long)C * D, 256), 256, 0, s>>>(C, D, state + Lo.m2, u);
  k_laps_state_init<<<1, 256, 0, s>>>(D, save_num, state);
  BJX_CHECK_LAUNCH("k_laps_init");
  return 0;
}

extern "C" int bjx_laps_burn_in_step(bjx_handle_t h, const uint32_t* phase_key, int32_t t, int32_t num_steps, float* q,
                                     float* u, float* logp, float* grad, float* state, const bjx_laps_burn_in_config* cfg,
                                     float* info) {
  const void* ptrs[] = {q, u, grad, state};
  int rc = check_ready(h, true, ptrs, 4);
  if (rc) return rc;
  if (!phase_key || !logp || !cfg) return bjx_fail(h, BJX_E_INVALID, "null argument");
  if (t < 0 || t >= num_steps) return bjx_fail(h, BJX_E_INVALID, "step index outside [0, num_steps)");
  if (cfg->bias_type < 0 || cfg->bias_type > 3) return bjx_fail(h, BJX_E_INVALID, "bias_type must be 0, 1, 2 or 3");
  if (cfg->bias_type == 2 && !cfg->equi_full)
    return bjx_fail(h, BJX_E_INVALID, "bias_type 2 needs equi_full (and a state sized with equi_full = 1)");
  if ((rc = laps_supported(h, cfg->save_num))) return rc;
  const int C = h->cfg.n_chains, D = h->cfg.dim;
  if ((long long)(h->chain_offset + (long long)C) * num_steps > 0xFFFFFFFFLL)
    return bjx_fail(h, BJX_E_INVALID, "n_chains * num_steps must be below 2^32 (split(key, (N, T)))");
  const bool equi = cfg->equi_full != 0;
  const Layout Lo(C, D, cfg->save_num, equi ? 1 : 0);
  const cudaStream_t s = h->stream;
  const Key pk{phase_key[0], phase_key[1]};
  const Key ks = fold_in(pk, 0u), kt = fold_in(fold_in(pk, 1u), (uint32_t)t);
  LaunchArgs a{};
  a.P = make_params(h, 0.f, nullptr);
  a.q_out = q;
  a.p_io = u;
  a.logp_out = logp;
  a.g_out = grad;
  a.laps.state = state;
  a.laps.rec = state + Lo.rec1;
  a.laps.key_a = ks.a;
  a.laps.key_b = ks.b;
  a.laps.T = (uint32_t)num_steps;
  a.laps.t = (uint32_t)t;
  if ((rc = dispatch(h, K_LAPS_BURN_IN, true, a))) return rc;
  merge(laps_grid(C), 3 * D + 4, state + Lo.rec1, state + Lo.part1, state + Lo.m1, state, s);
  if (equi) {
    const int chunks = zgx_chunks(C);
    k_laps_rademacher<<<blocks_for(kZRows * D, 256), 256, 0, s>>>(D, kt.a, kt.b, state + Lo.z, state);
    k_laps_zg<<<blocks_for(C, 8), 256, 0, s>>>(C, D, state + Lo.z, grad, state + Lo.a, state);
    k_laps_zgx<<<dim3(blocks_for(D, 128), chunks), 128, 0, s>>>(C, D, state + Lo.a, q, state + Lo.bp, state);
    k_laps_equi_full<<<1, kUpd, 0, s>>>(C, D, chunks, state + Lo.z, state + Lo.bp, state);
  }
  BurnInUpdate U{C, D, cfg->save_num, cfg->bias_type, cfg->early_stop ? 1 : 0, t, cfg->alpha, cfg->C, cfg->r_end};
  k_laps_update<<<1, kUpd, 0, s>>>(U, state + Lo.m1, state, info);
  BJX_CHECK_LAUNCH("k_laps_update");
  return 0;
}

extern "C" int bjx_laps_burn_in_run(bjx_handle_t h, const uint32_t* phase_key, int32_t num_steps, float* q, float* u,
                                    float* logp, float* grad, float* state, const bjx_laps_burn_in_config* cfg,
                                    float* info, int32_t chunk, int32_t* steps_run) {
  if (!h || !steps_run || num_steps < 0 || chunk < 1) return bjx_fail(h, BJX_E_INVALID, "bad argument");
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  int* pinned = nullptr;
  BJX_CUDA(cudaMallocHost(&pinned, 2 * sizeof(int)));
  struct Free {
    int* p;
    ~Free() { cudaFreeHost(p); }
  } guard{pinned};
  int rc = 0;
  for (int t = 0; t < num_steps && rc == 0; ++t) {
    rc = bjx_laps_burn_in_step(h, phase_key, t, num_steps, q, u, logp, grad, state, cfg, info);
    if (rc == 0 && cfg->early_stop && ((t + 1) % chunk == 0) && t + 1 < num_steps) {
      BJX_CUDA(cudaMemcpyAsync(pinned, reinterpret_cast<int*>(state) + LS_STOP, sizeof(int), cudaMemcpyDeviceToHost,
                               h->stream));
      BJX_CUDA(cudaStreamSynchronize(h->stream));
      if (pinned[0]) break;
    }
  }
  if (rc) return rc;
  if (num_steps == 0) {
    *steps_run = 0;
    return 0;
  }
  BJX_CUDA(cudaMemcpyAsync(pinned + 1, reinterpret_cast<int*>(state) + LS_COUNT, sizeof(int), cudaMemcpyDeviceToHost,
                           h->stream));
  BJX_CUDA(cudaStreamSynchronize(h->stream));
  *steps_run = pinned[1];
  return 0;
}

extern "C" int bjx_laps_switch(bjx_handle_t h, float* state, int32_t diagonal_preconditioning) {
  const void* ptrs[] = {state};
  int rc = check_ready(h, false, ptrs, 1);
  if (rc) return rc;
  k_laps_switch<<<1, kUpd, 0, h->stream>>>(h->cfg.dim, diagonal_preconditioning ? 1 : 0, state);
  BJX_CHECK_LAUNCH("k_laps_switch");
  return 0;
}

extern "C" int bjx_laps_adjusted_step(bjx_handle_t h, const uint32_t* phase_key, int32_t t, int32_t num_samples, float* q,
                                      float* logp, float* grad, float* state, int32_t save_num, int32_t steps_per_sample,
                                      float target_acceptance, int32_t diagnostics, float* info) {
  const void* ptrs[] = {q, grad, state};
  int rc = check_ready(h, true, ptrs, 3);
  if (rc) return rc;
  if (!phase_key || !logp || steps_per_sample < 0) return bjx_fail(h, BJX_E_INVALID, "bad argument");
  if (t < 0 || t >= num_samples) return bjx_fail(h, BJX_E_INVALID, "step index outside [0, num_samples)");
  if ((rc = laps_supported(h, save_num))) return rc;
  const int C = h->cfg.n_chains, D = h->cfg.dim;
  if ((long long)(h->chain_offset + (long long)C) * num_samples > 0xFFFFFFFFLL)
    return bjx_fail(h, BJX_E_INVALID, "n_chains * num_samples must be below 2^32 (split(key, (N, T)))");
  const Layout Lo(C, D, save_num, 0);  // the phase-2 regions lie within either sizing
  const cudaStream_t s = h->stream;
  const Key ks = fold_in(Key{phase_key[0], phase_key[1]}, 0u);
  uint32_t* keys = reinterpret_cast<uint32_t*>(state + Lo.keys);
  float* eps = state + Lo.eps;
  float* acc = state + Lo.acc;
  k_laps_keys<<<blocks_for(C, 256), 256, 0, s>>>(C, ks.a, ks.b, h->chain_offset, (uint32_t)num_samples, (uint32_t)t, keys);
  launch_fill_from(C, state + LS_EPS, eps, s);
  BJX_CHECK_LAUNCH("k_laps_keys");
  LaunchArgs a{};
  a.P = make_params(h, 0.f, eps);
  a.P.key_shared = 0;
  a.P.div_thr = 1000.f;
  a.keys = keys;
  a.q_in = q;
  a.logp_in = logp;
  a.g_in = grad;
  a.q_out = q;
  a.logp_out = logp;
  a.g_out = grad;
  a.amclmc.L_factor = 1.25f;
  a.amclmc.n = steps_per_sample;
  a.amclmc.rule = AMCLMC_STEPS_FIXED;
  a.info.acceptance_rate = acc;
  if ((rc = dispatch(h, K_AMCLMC, true, a))) return rc;
  k_laps_rowstats<<<stat_grid(C), 256, 0, s>>>(C, D, q, grad, acc, diagnostics ? 1 : 0, state + Lo.rec2);
  merge(stat_grid(C), D + 1, state + Lo.rec2, state + Lo.part2, state + Lo.m2, nullptr, s);
  k_laps_bisect<<<1, kUpd, 0, s>>>(C, D, diagnostics ? 1 : 0, state + Lo.m2, target_acceptance, steps_per_sample, t, state,
                                   info);
  BJX_CHECK_LAUNCH("k_laps_bisect");
  return 0;
}

extern "C" int bjx_laps_adjusted_run(bjx_handle_t h, const uint32_t* phase_key, int32_t num_samples, float* q, float* logp,
                                     float* grad, float* state, int32_t save_num, int32_t steps_per_sample,
                                     float target_acceptance, int32_t diagnostics, float* info) {
  if (!h || num_samples < 0) return bjx_fail(h, BJX_E_INVALID, "bad argument");
  int rc = 0;
  for (int t = 0; t < num_samples && rc == 0; ++t)
    rc = bjx_laps_adjusted_step(h, phase_key, t, num_samples, q, logp, grad, state, save_num, steps_per_sample,
                                target_acceptance, diagnostics, info);
  return rc;
}
