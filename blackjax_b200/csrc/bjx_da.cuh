// Dual averaging of the log step size (optimizers/dual_averaging.py:87-129, adaptation/step_size.py:65-150) on one
// 5-float state (log_step, log_step_avg, step, avg_error, mu).  Every warm-up on the device goes through these: the
// per-chain kernels (bjx_misc.cu), the pooled window recipes (bjx_pooled_step.cuh), ChEES (bjx_adapt.cu) and adjusted
// MCLMC's fused tuning step (bjx_kernels.cuh).
#pragma once

namespace bjx {

// dual_averaging.py:87-99 at the step size eps0: mu = log(10 eps0)
__device__ __forceinline__ void da_init(float* s, float eps0) {
  s[0] = logf(eps0);
  s[1] = 0.f;
  s[2] = 1.f;
  s[3] = 0.f;
  s[4] = logf(10.f * eps0);
}

// dual_averaging.py:101-123 with t0 = 10, gamma = 0.05, kappa = 0.75: updates s[0], s[1], s[2], s[3] in place
__device__ __forceinline__ void da_update_step(float* s, float acceptance_rate, float target) {
  const float log_step = s[0], avg_log_step = s[1], step = s[2];
  float avg_error = s[3];
  const float mu = s[4];
  const float gradient = target - acceptance_rate;
  const float reg_step = step + 10.f;                    // t0 = 10
  const float eta_t = powf(step, -0.75f);                // kappa = 0.75
  avg_error = (1.f - (1.f / reg_step)) * avg_error + gradient / reg_step;
  const float log_x = mu - (sqrtf(step) / 0.05f) * avg_error;  // gamma = 0.05
  const float log_x_avg = eta_t * log_step + (1.f - eta_t) * avg_log_step;  // uses the PRE-update iterate (:122)
  s[0] = log_x;
  s[1] = log_x_avg;
  s[2] = step + 1.f;
  s[3] = avg_error;
}

// the step size the next transition uses, and the one a warm-up returns (the averaged iterate)
__device__ __forceinline__ float da_step_size(const float* s) { return expf(s[0]); }
__device__ __forceinline__ float da_final(const float* s) { return expf(s[1]); }

// a window end (staged_adaptation.py:233-249): a fresh state at the averaged step size
__device__ __forceinline__ void da_restart(float* s) { da_init(s, da_final(s)); }

}  // namespace bjx
