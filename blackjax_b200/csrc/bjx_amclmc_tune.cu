// Adjusted MCLMC's tuner (blackjax/adaptation/adjusted_mclmc_adaptation.py:26-507): one fused tuning step and
// adjusted_mclmc_find_L_and_step_size run on the device with no host synchronisation.  Chains never interact: every chain
// runs the reference's single-chain tuner with its own key, as jax.vmap over chains would.
//
// Key tree of chain c, whose key k_c is split(rng_key, n_global)[chain_offset + c] or the caller's per-chain key:
//   part1, part2 = split(k_c)                                                                   :128
//   window i: window_key = fold_in(part1, i); check, rk = split(window_key); p1, p2 = split(rk)  :132, :332-334
//     pass-1 step t: split(p1, n1 + n2)[t];  pass-2 step t: split(p2, n1)[t]                    :335-338
//   stage 3, window i: part2 = fold_in(part2, i) (cumulative); k1, k2 = split(part2)             :156-157
//     transition t: split(k1, n3)[t];  the adaptation that follows: the window tree from k2     :446, :193
// split(key, n)[i] = fold_in(key, i), so every step key comes from its parent key and index (bjx_mclmc_tune.cu).
#include <math.h>

#include "../../include/bjx.h"
#include "bjx_internal.h"
#include "bjx_launch.cuh"
#include "bjx_handle.h"

using namespace bjx;

namespace {

// L = target_k * step_size: the entry and exit pins (:126, :203) and the re-pin before pass 2 (:412-414)
__global__ void k_atune_pin(int C, float target_k, const float* __restrict__ eps, float* __restrict__ L) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) L[c] = __fmul_rn(target_k, eps[c]);
}

// each scan's fresh state: streaming (total, average) = (0, 0) (:322); count untouched
__global__ void k_atune_reset(int C, float* __restrict__ total) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) total[c] = 0.f;
}

// the window keys: p1[c], p2[c] = split(split(fold_in(base[c], i))[1])
__global__ void k_atune_window_keys(int C, const uint32_t* __restrict__ base, uint32_t i, uint32_t* __restrict__ p1,
                                    uint32_t* __restrict__ p2) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const Key rk = fold_in(fold_in(Key{base[2 * c], base[2 * c + 1]}, i), 1u);
  const Key a = fold_in(rk, 0u), b = fold_in(rk, 1u);
  p1[2 * c] = a.a;
  p1[2 * c + 1] = a.b;
  p2[2 * c] = b.a;
  p2[2 * c + 1] = b.b;
}

// after pass 1, if n2 != 0 (:373-414): var = E[x^2] - E[x]^2, change = clamp(0, contract(var) / L, 2) with contract
// sqrt(sum var) * tuning_factor (max = 0) or sqrt(max var * D) * tuning_factor (max = 1); step *= change; with diagonal
// preconditioning M^-1 = var; then L = target_k * step (the rescaled L is overwritten by the re-pin).  One warp per chain.
__global__ void k_atune_variance(int C, int D, const float* __restrict__ moments, int diag, int use_max,
                                 float tuning_factor, float target_k, float* __restrict__ imm, float* __restrict__ eps,
                                 float* __restrict__ L) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (c >= C) return;
  const float* m1 = moments + (size_t)c * 2 * D;
  const float* m2 = m1 + D;
  float acc = use_max ? -__int_as_float(0x7f800000) : 0.f;
  for (int d = lane; d < D; d += 32) {
    const float v = __fsub_rn(m2[d], __fmul_rn(m1[d], m1[d]));
    acc = use_max ? fmaxf(acc, v) : __fadd_rn(acc, v);
    if (diag) imm[(size_t)c * D + d] = v;
  }
  if (use_max) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc = fmaxf(acc, __shfl_xor_sync(0xffffffffu, acc, o));
  } else {
    acc = warp_sum(acc);
  }
  if (lane == 0) {
    const float contract = __fmul_rn(sqrtf(use_max ? __fmul_rn(acc, (float)D) : acc), tuning_factor);
    const float change = fminf(fmaxf(__fdiv_rn(contract, L[c]), 0.f), 2.f);
    const float e = __fmul_rn(eps[c], change);
    eps[c] = e;
    L[c] = __fmul_rn(target_k, e);
  }
}

// stage 3's step-count argument, avg = L / step_size per chain (:455)
__global__ void k_atune_avg(int C, const float* __restrict__ L, const float* __restrict__ eps, float* __restrict__ avg) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) avg[c] = __fdiv_rn(L[c], eps[c]);
}

// stage 3 (:465-486): r = contract_d(ESS) / n3 (mean, or min for max = 1), L = min(l_factor * L / r, 2 L).  One warp per
// chain.
__global__ void k_atune_L_from_ess(int C, int D, int n3, const float* __restrict__ ess, int use_max, float l_factor,
                                   float* __restrict__ L) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (c >= C) return;
  float acc = use_max ? __int_as_float(0x7f800000) : 0.f;
  for (int d = lane; d < D; d += 32) {
    const float e = ess[(size_t)c * D + d];
    acc = use_max ? fminf(acc, e) : __fadd_rn(acc, e);
  }
  if (use_max) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc = fminf(acc, __shfl_xor_sync(0xffffffffu, acc, o));
  } else {
    acc = __fdiv_rn(warp_sum(acc), (float)D);
  }
  if (lane == 0) {
    const float r = __fdiv_rn(acc, (float)n3);
    const float l = L[c];
    L[c] = fminf(__fdiv_rn(__fmul_rn(l_factor, l), r), __fmul_rn(l, 2.0f));
  }
}

int tune_dispatch(bjx_handle_t h, const Params& P, const uint32_t* keys, float* q, float* logp, float* grad,
                  const AmclmcTuneArgs& T) {
  LaunchArgs a{};
  a.P = P;
  a.keys = keys;
  a.q_out = q;
  a.logp_out = logp;
  a.g_out = grad;
  a.amclmc_tune = T;
  return dispatch(h, K_AMCLMC_TUNE, true, a);
}

int check_rule(bjx_handle_t h, const uint32_t* random_generator_arg, int steps_rule) {
  if (random_generator_arg && (steps_rule < BJX_AMCLMC_STEPS_FIXED || steps_rule > BJX_AMCLMC_STEPS_UNIFORM))
    return bjx_fail(h, BJX_E_INVALID, "unknown steps_rule");
  return 0;
}

}  // namespace

extern "C" int bjx_adjusted_mclmc_tune_step(bjx_handle_t h, const uint32_t* keys, float* q, float* logp, float* grad,
                                            uint32_t* random_generator_arg, int32_t steps_rule, int32_t min_steps,
                                            float* step_size, float* L, float* da_state, float* total, float* moments,
                                            float* count, int32_t mask, int32_t fix_L, float target, uint8_t* success,
                                            int32_t* steps) {
  const void* ptrs[] = {q, grad};
  int rc = check_ready(h, true, ptrs, 2);
  if (rc) return rc;
  if (!keys || !logp || !step_size || !L || !da_state || (!mask && moments && !total))
    return bjx_fail(h, BJX_E_INVALID, "null argument");
  if (moments && size_class_is_vec(h->sc) && ((uintptr_t)moments & 15u))
    return bjx_fail(h, BJX_E_INVALID, "moments must be 16-byte aligned");
  if ((rc = check_rule(h, random_generator_arg, steps_rule))) return rc;
  if ((rc = mclmc_transition_supported(h, "adjusted MCLMC tuning"))) return rc;
  AmclmcTuneArgs T{};
  T.eps = step_size;
  T.L = L;
  T.da = da_state;
  T.total = total;
  T.moments = moments;
  T.count = count;
  T.rga = random_generator_arg;
  T.rule = steps_rule;
  T.min_steps = min_steps;
  T.mask = mask ? 1 : 0;
  T.fix_L = fix_L ? 1 : 0;
  T.target = target;
  T.success = success;
  T.steps = steps;
  return tune_dispatch(h, make_params(h, 0.f, nullptr), keys, q, logp, grad, T);
}

extern "C" int bjx_adjusted_mclmc_find_l_and_step_size(
    bjx_handle_t h, const uint32_t* rng_key, float* q, float* logp, float* grad, uint32_t* random_generator_arg,
    int32_t steps_rule, int32_t min_steps, float* step_size, float* L, float* inverse_mass_matrix, int32_t num_windows,
    int32_t num_steps1, int32_t num_steps2, int32_t num_steps3, float target, int32_t diagonal_preconditioning,
    int32_t use_max, float tuning_factor, float target_num_integration_steps, double l_factor,
    int64_t max_history_bytes, float* num_integration_steps) {
  const void* ptrs[] = {q, grad, inverse_mass_matrix};
  int rc = check_ready(h, true, ptrs, 3);
  if (rc) return rc;
  if (!rng_key || !logp || !step_size || !L || !num_integration_steps) return bjx_fail(h, BJX_E_INVALID, "null argument");
  if (num_windows < 0 || num_steps1 < 0 || num_steps2 < 0 || num_steps3 < 0 || max_history_bytes < 0)
    return bjx_fail(h, BJX_E_INVALID, "negative window count, stage length or history budget");
  if (num_steps3 == 1) return bjx_fail(h, BJX_E_INVALID, "The input array must have at least 2 samples");
  if ((rc = check_rule(h, random_generator_arg, steps_rule))) return rc;
  if ((rc = mclmc_transition_supported(h, "adjusted MCLMC tuning"))) return rc;
  const int C = h->cfg.n_chains, D = h->cfg.dim;
  const cudaStream_t st = h->stream;
  const bool stage3 = num_steps3 >= 2;
  // stage 3 runs on slices of cs chains whose position history [n3, cs, D] fits the budget (at least one chain)
  const long long cs = stage3 ? history_slice_chains(max_history_bytes, num_steps3, D, C) : 1;
  // scratch: part1, part2, p1, p2, step keys [C, 2] u32 | da [C, 5] | total, avg [C] | moments [C, 2, D] |
  // history [n3, cs, D] | ess [cs, D]; float offsets rounded up to 4 floats keep every row 16-byte aligned
  auto up4 = [](size_t n) { return (n + 3) & ~(size_t)3; };
  const size_t o_da = up4(10 * (size_t)C), o_scal = o_da + up4(5 * (size_t)C), o_mom = o_scal + up4(2 * (size_t)C);
  const size_t o_hist = o_mom + 2 * (size_t)C * D;
  const size_t o_ess = o_hist + (stage3 ? (size_t)num_steps3 * cs * D : 0), n_floats = o_ess + (stage3 ? cs * D : 0);
  StreamScratch scratch(h);
  BJX_CUDA(cudaMallocAsync(&scratch.ptr, n_floats * sizeof(float), st));
  float* ws = static_cast<float*>(scratch.ptr);
  uint32_t* part1 = reinterpret_cast<uint32_t*>(ws);
  uint32_t* part2 = part1 + 2 * (size_t)C;
  uint32_t* p1 = part2 + 2 * (size_t)C;
  uint32_t* p2 = p1 + 2 * (size_t)C;
  uint32_t* step_keys = p2 + 2 * (size_t)C;
  float* da = ws + o_da;
  float* total = ws + o_scal;
  float* avg = total + C;
  float* moments = ws + o_mom;
  float* history = ws + o_hist;
  float* ess = ws + o_ess;

  BJX_CUDA(cudaMemsetAsync(num_integration_steps, 0, sizeof(float) * C, st));
  launch_tune_part_keys(C, h->key_shared, h->chain_offset, rng_key, part1, part2, st);
  BJX_CHECK_LAUNCH("k_tune_part_keys");
  k_atune_pin<<<blocks_for(C, 256), 256, 0, st>>>(C, target_num_integration_steps, step_size, L);  // entry pin
  BJX_CHECK_LAUNCH("k_atune_pin");
  Params P = make_params(h, 0.f, step_size);
  P.imm = inverse_mass_matrix;  // the tuner's own per-chain diagonal metric
  P.imm_stride = D;
  P.imm_group = 1;
  P.key_shared = 0;
  AmclmcTuneArgs T{};
  T.eps = step_size;
  T.L = L;
  T.da = da;
  T.total = total;
  T.moments = moments;
  T.count = num_integration_steps;
  T.rga = random_generator_arg;
  T.rule = steps_rule;
  T.min_steps = min_steps;
  T.target = target;
  // one step_size_adaptation scan (:315-325): a fresh dual averaging from the current step size, n steps with keys
  // split(base, n)[t], masked in (m = 1) for t < n_masked; then step_size = final_da (:368-369, :432)
  auto pass = [&](const uint32_t* base, int n, int n_masked, bool fix_L) -> int {
    launch_da(0, C, da, step_size, 0.f, nullptr, st);
    BJX_CHECK_LAUNCH("k_da_init");
    k_atune_reset<<<blocks_for(C, 256), 256, 0, st>>>(C, total);
    BJX_CHECK_LAUNCH("k_atune_reset");
    if (n > n_masked) BJX_CUDA(cudaMemsetAsync(moments, 0, sizeof(float) * 2 * (size_t)C * D, st));
    T.fix_L = fix_L ? 1 : 0;
    for (int t = 0; t < n; ++t) {
      launch_tune_fold_keys(C, base, (uint32_t)t, step_keys, st);
      BJX_CHECK_LAUNCH("k_tune_fold_keys");
      T.mask = t < n_masked ? 1 : 0;
      int r = tune_dispatch(h, P, step_keys, q, logp, grad, T);
      if (r) return r;
    }
    launch_da(3, C, da, nullptr, 0.f, step_size, st);
    BJX_CHECK_LAUNCH("k_da_final");
    return 0;
  };
  // adjusted_mclmc_make_L_step_size_adaptation (:327-434) from the window key fold_in(base, i)
  auto window = [&](const uint32_t* base, uint32_t i, int n2) -> int {
    k_atune_window_keys<<<blocks_for(C, 256), 256, 0, st>>>(C, base, i, p1, p2);
    BJX_CHECK_LAUNCH("k_atune_window_keys");
    int r = pass(p1, num_steps1 + n2, num_steps1, true);  // pass 1, fix_L (:351-365)
    if (r || n2 == 0) return r;
    k_atune_variance<<<blocks_for(C, kWarpsPerBlock), kThreads, 0, st>>>(
        C, D, moments, diagonal_preconditioning ? 1 : 0, use_max ? 1 : 0, tuning_factor, target_num_integration_steps,
        inverse_mass_matrix, step_size, L);
    BJX_CHECK_LAUNCH("k_atune_variance");
    return pass(p2, num_steps1, num_steps1, false);  // pass 2 (:416-432)
  };
  for (int i = 0; i < num_windows; ++i)
    if ((rc = window(part1, (uint32_t)i, num_steps2))) return rc;
  if (stage3) {
    for (int i = 0; i < num_windows; ++i) {
      launch_tune_fold_keys(C, part2, (uint32_t)i, part2, st);  // part2 = fold_in(part2, i)
      BJX_CHECK_LAUNCH("k_tune_fold_keys");
      launch_tune_fold_keys(C, part2, 0u, p1, st);  // k1; p1 is free until the window below
      BJX_CHECK_LAUNCH("k_tune_fold_keys");
      k_atune_avg<<<blocks_for(C, 256), 256, 0, st>>>(C, L, step_size, avg);
      BJX_CHECK_LAUNCH("k_atune_avg");
      // adjusted_mclmc_make_adaptation_L (:444-489), one slice of chains at a time
      auto step = [&](long long c0, int n, int t) -> int {
        const size_t row = (size_t)c0 * D;
        LaunchArgs a{};
        a.P = P;
        a.P.C = n;
        a.P.imm = inverse_mass_matrix + row;
        a.P.eps_dev = step_size + c0;
        a.keys = step_keys;
        a.q_in = a.q_out = q + row;
        a.logp_in = a.logp_out = logp + c0;
        a.g_in = a.g_out = grad + row;
        a.amclmc.L_factor = INFINITY;
        a.amclmc.rule = random_generator_arg ? steps_rule : BJX_AMCLMC_STEPS_FIXED;
        a.amclmc.min_steps = random_generator_arg ? min_steps : 0;
        a.amclmc.rga = random_generator_arg ? random_generator_arg + 2 * c0 : nullptr;
        a.amclmc.avg = avg + c0;
        a.amclmc.count = num_integration_steps + c0;
        a.amclmc.count_avg = random_generator_arg ? 0 : 1;
        launch_tune_fold_keys(n, p1 + 2 * c0, (uint32_t)t, step_keys, st);
        BJX_CHECK_LAUNCH("k_tune_fold_keys");
        return dispatch(h, K_AMCLMC, true, a);
      };
      auto finish = [&](long long c0, int n) -> int {
        k_atune_L_from_ess<<<blocks_for(n, kWarpsPerBlock), kThreads, 0, st>>>(n, D, num_steps3, ess, use_max ? 1 : 0,
                                                                               (float)l_factor, L + c0);
        BJX_CHECK_LAUNCH("k_atune_L_from_ess");
        return 0;
      };
      if ((rc = run_ess_slices(h, cs, num_steps3, q, history, ess, step, finish))) return rc;
      // the pass-1-only adaptation from k2 = split(part2)[1] (:176-194): its window key is k2 itself, so fold_in(part2,
      // 1) stands in for fold_in(base, i)
      if ((rc = window(part2, 1u, 0))) return rc;
    }
  }
  k_atune_pin<<<blocks_for(C, 256), 256, 0, st>>>(C, target_num_integration_steps, step_size, L);  // exit pin
  BJX_CHECK_LAUNCH("k_atune_pin");
  return 0;
}

// The step count of a rule for every chain from its random_generator_arg (not advanced) and per-chain avg.
__global__ void k_amclmc_num_steps(int C, int rule, const float* __restrict__ avg, int min_steps,
                                   const uint32_t* __restrict__ rga, int32_t* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float a = avg ? avg[c] : 0.f;
  const float scale = rule == AMCLMC_STEPS_UNIFORM ? amclmc_rescale(a) : 0.f;
  out[c] = amclmc_rule_steps(rule, rga ? rga + 2 * c : nullptr, a, scale, min_steps);
}

extern "C" int bjx_adjusted_mclmc_num_steps(bjx_handle_t h, int32_t steps_rule, const float* avg, int32_t min_steps,
                                            const uint32_t* random_generator_arg, int32_t* steps_out) {
  if (!h || !steps_out) return bjx_fail(h, BJX_E_INVALID, "null argument");
  if (steps_rule < BJX_AMCLMC_STEPS_FIXED || steps_rule > BJX_AMCLMC_STEPS_UNIFORM)
    return bjx_fail(h, BJX_E_INVALID, "unknown steps_rule");
  if ((steps_rule != BJX_AMCLMC_STEPS_RANDINT && !avg) || (steps_rule != BJX_AMCLMC_STEPS_FIXED && !random_generator_arg))
    return bjx_fail(h, BJX_E_INVALID, "the rule needs avg and, unless fixed, random_generator_arg");
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  const int C = h->cfg.n_chains;
  k_amclmc_num_steps<<<blocks_for(C, 256), 256, 0, h->stream>>>(C, steps_rule, avg, min_steps, random_generator_arg,
                                                                steps_out);
  BJX_CHECK_LAUNCH("k_amclmc_num_steps");
  return 0;
}
