// MCLMC's L / step-size tuner (blackjax/adaptation/mclmc_adaptation.py:42-399): one fused tuning step, the per-chain ESS,
// and the three stages of mclmc_find_L_and_step_size run on the device with no host synchronisation.  Chains never
// interact: every chain runs the reference's single-chain tuner with its own key, as jax.vmap over chains would.
//
// Key tree of chain c, whose key k_c is split(rng_key, n_global)[chain_offset + c] or the caller's per-chain key:
//   part1, part2 = split(k_c)                                                               :177
//   stage 1 and 2 step t: split(part1, n1 + n2 + 1)[t];  final_key = [n1 + n2]              :322-328
//   readjust step t: split(final_key, r)[t]                                                 :357
//   stage 3 step t: split(part2, n3)[t], the plain transition's key                         :372
// split(key, n)[i] = fold_in(key, i), so every step key comes from its part key and index; no [T, C, 2] array exists.
#include <math.h>

#include "../../include/bjx.h"
#include "bjx_internal.h"
#include "bjx_launch.cuh"
#include "bjx_handle.h"

using namespace bjx;

namespace {

// part1[c], part2[c] = split(k_c)
__global__ void k_tune_part_keys(int C, int key_shared, uint32_t chain_offset, const uint32_t* __restrict__ keys,
                                 uint32_t* __restrict__ part1, uint32_t* __restrict__ part2) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const Key k = key_shared ? fold_in(Key{keys[0], keys[1]}, chain_offset + (uint32_t)c) : Key{keys[2 * c], keys[2 * c + 1]};
  const Key a = fold_in(k, 0u), b = fold_in(k, 1u);
  part1[2 * c] = a.a;
  part1[2 * c + 1] = a.b;
  part2[2 * c] = b.a;
  part2[2 * c + 1] = b.b;
}

// out[c] = split(base[c], n)[i]
__global__ void k_tune_fold_keys(int C, const uint32_t* base, uint32_t i, uint32_t* out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const Key k = fold_in(Key{base[2 * c], base[2 * c + 1]}, i);
  out[2 * c] = k.a;
  out[2 * c + 1] = k.b;
}

// the scan's initial adaptive state (time, x_average, step_size_max) = (0, 0, inf) and streaming weight 0 (:307-311)
__global__ void k_tune_reset(int C, float* time, float* x_avg, float* eps_max, float* total) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  time[c] = 0.f;
  x_avg[c] = 0.f;
  eps_max[c] = __int_as_float(0x7f800000);
  total[c] = 0.f;
}

// after stages 1 and 2 (:340-353): var = E[x^2] - E[x]^2 (unclamped), L = sqrt(sum var); with diagonal preconditioning
// M^-1 = var and L = sqrt(D).  One warp per chain.
__global__ void k_tune_variance(int C, int D, const float* __restrict__ moments, int diag, float* __restrict__ imm,
                                float* __restrict__ L_out) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (c >= C) return;
  const float* m1 = moments + (size_t)c * 2 * D;
  const float* m2 = m1 + D;
  float acc = 0.f;
  for (int d = lane; d < D; d += 32) {
    const float v = __fsub_rn(m2[d], __fmul_rn(m1[d], m1[d]));
    acc = __fadd_rn(acc, v);
    if (diag) imm[(size_t)c * D + d] = v;
  }
  acc = warp_sum(acc);
  if (lane == 0) L_out[c] = diag ? sqrtf((float)D) : sqrtf(acc);
}

// stage 3 (:393-397): L = l_factor * eps * mean_d(n3 / ess[c, d]); a dimension with ESS 0 makes L = inf.  One warp per chain.
__global__ void k_tune_L_from_ess(int C, int D, int n3, const float* __restrict__ ess, const float* __restrict__ eps,
                                  float l_factor, float* __restrict__ L_out) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (c >= C) return;
  float acc = 0.f;
  for (int d = lane; d < D; d += 32) acc = __fadd_rn(acc, __fdiv_rn((float)n3, ess[(size_t)c * D + d]));
  acc = warp_sum(acc);
  if (lane == 0) L_out[c] = __fmul_rn(__fmul_rn(l_factor, eps[c]), __fdiv_rn(acc, (float)D));
}

// the predictor's constants as the reference forms them: Python floats (double), then float32 in the jnp expressions
struct TuneConstants {
  float dim_eev, trust6, decay;
};
TuneConstants tune_constants(int D, double desired_energy_var, double trust_in_estimate, double num_effective_samples) {
  return {(float)((double)D * desired_energy_var), (float)(6.0 * trust_in_estimate),
          (float)((num_effective_samples - 1.0) / (num_effective_samples + 1.0))};
}

int tune_dispatch(bjx_handle_t h, const Params& P, const uint32_t* keys, float* q, float* p, float* logp, float* grad,
                  const MclmcTuneArgs& T) {
  LaunchArgs a{};
  a.P = P;
  a.keys = keys;
  a.q_out = q;
  a.p_io = p;
  a.logp_out = logp;
  a.g_out = grad;
  a.mclmc_tune = T;
  return dispatch(h, K_MCLMC_TUNE, true, a);
}

}  // namespace

namespace bjx {
void launch_tune_part_keys(int C, int key_shared, uint32_t chain_offset, const uint32_t* keys, uint32_t* part1,
                           uint32_t* part2, cudaStream_t s) {
  k_tune_part_keys<<<blocks_for(C, 256), 256, 0, s>>>(C, key_shared, chain_offset, keys, part1, part2);
}
void launch_tune_fold_keys(int C, const uint32_t* base, uint32_t i, uint32_t* out, cudaStream_t s) {
  k_tune_fold_keys<<<blocks_for(C, 256), 256, 0, s>>>(C, base, i, out);
}
}  // namespace bjx

extern "C" int bjx_mclmc_tune_step(bjx_handle_t h, const uint32_t* keys, float* q, float* p, float* logp, float* grad,
                                   float* step_size, float L, const float* L_dev, float energy_cutoff, float* time,
                                   float* x_average, float* step_size_max, float* total, float* moments, int32_t mask,
                                   double desired_energy_var, double trust_in_estimate, double num_effective_samples,
                                   uint8_t* success) {
  const void* ptrs[] = {q, p, grad};
  int rc = check_ready(h, true, ptrs, 3);
  if (rc) return rc;
  if (!keys || !logp || !step_size || !time || !x_average || !step_size_max || (mask && moments && !total))
    return bjx_fail(h, BJX_E_INVALID, "null argument");
  if (moments && size_class_is_vec(h->sc) && ((uintptr_t)moments & 15u))
    return bjx_fail(h, BJX_E_INVALID, "moments must be 16-byte aligned");
  if ((rc = mclmc_transition_supported(h, "MCLMC tuning"))) return rc;
  const TuneConstants k = tune_constants(h->cfg.dim, desired_energy_var, trust_in_estimate, num_effective_samples);
  MclmcTuneArgs T{};
  T.m.L = L;
  T.m.L_dev = L_dev;
  T.m.energy_cutoff = energy_cutoff;
  T.eps = step_size;
  T.time = time;
  T.x_avg = x_average;
  T.eps_max = step_size_max;
  T.total = total;
  T.moments = moments;
  T.mask = mask ? 1 : 0;
  T.dim_eev = k.dim_eev;
  T.trust6 = k.trust6;
  T.decay = k.decay;
  T.success = success;
  return tune_dispatch(h, make_params(h, 0.f, nullptr), keys, q, p, logp, grad, T);
}

extern "C" int bjx_mclmc_ess_per_chain(bjx_handle_t h, const float* history, int32_t num_samples, float* ess_out,
                                       int32_t* lags_evaluated) {
  if (!h || !history || !ess_out) return bjx_fail(h, BJX_E_INVALID, "null argument");
  if (num_samples < 2) return bjx_fail(h, BJX_E_INVALID, "The input array must have at least 2 samples");
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  if (lags_evaluated) BJX_CUDA(cudaMemsetAsync(lags_evaluated, 0, sizeof(int32_t) * h->cfg.n_chains, h->stream));
  launch_ess_per_chain(num_samples, h->cfg.n_chains, h->cfg.dim, history, ess_out, lags_evaluated, h->stream);
  BJX_CHECK_LAUNCH("k_ess_chain");
  return 0;
}

extern "C" int bjx_mclmc_find_l_and_step_size(bjx_handle_t h, const uint32_t* rng_key, float* q, float* p, float* logp,
                                              float* grad, float* step_size, float* L, float* inverse_mass_matrix,
                                              int32_t num_steps1, int32_t num_steps2, int32_t readjust_steps,
                                              int32_t num_steps3, int32_t diagonal_preconditioning, float energy_cutoff,
                                              double desired_energy_var, double trust_in_estimate,
                                              double num_effective_samples, double l_factor, int64_t max_history_bytes,
                                              uint8_t* divergence_history) {
  const void* ptrs[] = {q, p, grad, inverse_mass_matrix};
  int rc = check_ready(h, true, ptrs, 4);
  if (rc) return rc;
  if (!rng_key || !logp || !step_size || !L) return bjx_fail(h, BJX_E_INVALID, "null argument");
  if (num_steps1 < 0 || num_steps2 < 0 || readjust_steps < 0 || num_steps3 < 0 || max_history_bytes < 0)
    return bjx_fail(h, BJX_E_INVALID, "negative stage length or history budget");
  if ((rc = mclmc_transition_supported(h, "MCLMC tuning"))) return rc;
  const int C = h->cfg.n_chains, D = h->cfg.dim;
  const cudaStream_t st = h->stream;
  const int n12 = num_steps1 + num_steps2;
  const bool estimate = num_steps2 > 1, readjust = estimate && diagonal_preconditioning && readjust_steps > 0;
  const bool stage3 = num_steps3 >= 2;
  // stage 3 runs on slices of cs chains whose position history [n3, cs, D] fits the budget (at least one chain)
  const long long cs = stage3 ? history_slice_chains(max_history_bytes, num_steps3, D, C) : 1;
  // scratch: part1, part2, step keys [C, 2] u32 | time, x_avg, eps_max, total, L_new [C] | moments [C, 2, D] |
  // history [n3, cs, D] | ess [cs, D]; float offsets rounded up to 4 floats keep every row 16-byte aligned
  auto up4 = [](size_t n) { return (n + 3) & ~(size_t)3; };
  const size_t o_scal = up4(6 * (size_t)C), o_mom = o_scal + up4(5 * (size_t)C), o_hist = o_mom + 2 * (size_t)C * D;
  const size_t o_ess = o_hist + (stage3 ? (size_t)num_steps3 * cs * D : 0), n_floats = o_ess + (stage3 ? cs * D : 0);
  StreamScratch scratch(h);
  BJX_CUDA(cudaMallocAsync(&scratch.ptr, n_floats * sizeof(float), st));
  float* ws = static_cast<float*>(scratch.ptr);
  uint32_t* part1 = reinterpret_cast<uint32_t*>(ws);
  uint32_t* part2 = part1 + 2 * (size_t)C;
  uint32_t* step_keys = part2 + 2 * (size_t)C;
  float* time = ws + o_scal;
  float *x_avg = time + C, *eps_max = x_avg + C, *total = eps_max + C, *L_new = total + C;
  float* moments = ws + o_mom;
  float* history = ws + o_hist;
  float* ess = ws + o_ess;

  k_tune_part_keys<<<blocks_for(C, 256), 256, 0, st>>>(C, h->key_shared, h->chain_offset, rng_key, part1, part2);
  BJX_CHECK_LAUNCH("k_tune_part_keys");
  Params P = make_params(h, 0.f, step_size);
  P.imm = inverse_mass_matrix;  // the tuner's own per-chain diagonal metric
  P.imm_stride = D;
  P.imm_group = 1;
  P.key_shared = 0;
  const TuneConstants k = tune_constants(D, desired_energy_var, trust_in_estimate, num_effective_samples);
  MclmcTuneArgs T{};
  T.m.L_dev = L;  // stages 1, 2 and the readjustment all run with the initial L
  T.m.energy_cutoff = energy_cutoff;
  T.eps = step_size;
  T.time = time;
  T.x_avg = x_avg;
  T.eps_max = eps_max;
  T.total = total;
  T.dim_eev = k.dim_eev;
  T.trust6 = k.trust6;
  T.decay = k.decay;
  auto run_steps = [&](const uint32_t* base, int n, int div_row0, bool accumulate) -> int {
    k_tune_reset<<<blocks_for(C, 256), 256, 0, st>>>(C, time, x_avg, eps_max, total);
    BJX_CHECK_LAUNCH("k_tune_reset");
    T.moments = accumulate ? moments : nullptr;
    for (int t = 0; t < n; ++t) {
      k_tune_fold_keys<<<blocks_for(C, 256), 256, 0, st>>>(C, base, (uint32_t)t, step_keys);
      BJX_CHECK_LAUNCH("k_tune_fold_keys");
      T.mask = accumulate && t >= num_steps1;  // the last num_steps2 steps estimate the moments (:331)
      T.diverged = divergence_history ? divergence_history + (size_t)(div_row0 + t) * C : nullptr;
      int r = tune_dispatch(h, P, step_keys, q, p, logp, grad, T);
      if (r) return r;
    }
    return 0;
  };
  // stages 1 and 2 (:322-336)
  BJX_CUDA(cudaMemsetAsync(moments, 0, sizeof(float) * 2 * (size_t)C * D, st));
  if ((rc = run_steps(part1, n12, 0, true))) return rc;
  if (estimate) {  // :340-360
    k_tune_variance<<<blocks_for(C, kWarpsPerBlock), kThreads, 0, st>>>(C, D, moments, diagonal_preconditioning ? 1 : 0,
                                                                        inverse_mass_matrix, L_new);
    BJX_CHECK_LAUNCH("k_tune_variance");
    if (readjust) {
      k_tune_fold_keys<<<blocks_for(C, 256), 256, 0, st>>>(C, part1, (uint32_t)n12, part1);  // part1 <- final_key
      BJX_CHECK_LAUNCH("k_tune_fold_keys");
      if ((rc = run_steps(part1, readjust_steps, n12, false))) return rc;
    }
    BJX_CUDA(cudaMemcpyAsync(L, L_new, sizeof(float) * C, cudaMemcpyDeviceToDevice, st));
  }
  if (!stage3) return 0;
  // stage 3 (:367-399), one slice of chains at a time: transitions, position history, per-chain ESS, L
  auto step = [&](long long c0, int n, int t) -> int {
    const size_t row = (size_t)c0 * D;
    LaunchArgs a{};
    a.P = P;
    a.P.C = n;
    a.P.imm = inverse_mass_matrix + row;
    a.P.eps_dev = step_size + c0;
    a.keys = step_keys;
    a.q_out = q + row;
    a.p_io = p + row;
    a.logp_out = logp + c0;
    a.g_out = grad + row;
    a.mclmc.L_dev = L + c0;
    a.mclmc.energy_cutoff = energy_cutoff;
    k_tune_fold_keys<<<blocks_for(n, 256), 256, 0, st>>>(n, part2 + 2 * c0, (uint32_t)t, step_keys);
    BJX_CHECK_LAUNCH("k_tune_fold_keys");
    return dispatch(h, K_MCLMC, true, a);
  };
  auto finish = [&](long long c0, int n) -> int {
    k_tune_L_from_ess<<<blocks_for(n, kWarpsPerBlock), kThreads, 0, st>>>(n, D, num_steps3, ess, step_size + c0,
                                                                          (float)l_factor, L + c0);
    BJX_CHECK_LAUNCH("k_tune_L_from_ess");
    return 0;
  };
  return run_ess_slices(h, cs, num_steps3, q, history, ess, step, finish);
}
