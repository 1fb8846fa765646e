// The step-size half of the pooled window recipes (bjx_adapt_shared_*, bjx_lowrank_window_*): ONE dual-averaging update
// per warm-up step on the mean acceptance rate of all chains (staged_adaptation.py:153-171), and the Chan-Golub-LeVeque
// scalar factors their merges share.
#pragma once
#include "bjx_da.cuh"

namespace bjx {

// slots 0-7 of a pooled state's header: the dual-averaging state, the step size the next transition uses, the count of
// the diagonal recipe's window accumulator (unused by the low-rank recipe) and the warm-up steps taken
enum { PS_DA = 0, PS_EPS = 5, PS_WINDOW_N = 6, PS_T = 7 };

// metric_buffers.py:334-393 with the reference's scalar arithmetic (exact integer counts, one rounding to float32)
__device__ __forceinline__ void cgl_factors(float na, float nb, float& f_mean, float& f_cross, float& n_ab) {
  const double ab = (double)na + (double)nb;
  n_ab = (float)ab;
  f_mean = (float)((double)nb / ab);
  f_cross = (float)((double)na * (double)nb / ab);
}

// One thread: sums (sum accept, n) over the nblk k_block_stats records (stride S) in global block order, takes the
// dual-averaging update on the mean acceptance rate, restarts it at a window end, stores the new step size in PS_EPS and
// eps_hist[t] (unless null) and bumps t.  Returns n, the chains of all blocks.
__device__ __forceinline__ float pooled_step_size_update(int nblk, const float* __restrict__ blocks, size_t S, float* __restrict__ st,
                                                         int window_end, float target, float* __restrict__ eps_hist) {
  float n = blocks[1], acc = blocks[0];
  for (int b = 1; b < nblk; ++b) {
    const float* g = blocks + (size_t)b * S;
    float fm, fc, nab;
    cgl_factors(n, g[1], fm, fc, nab);
    n = nab;
    acc += g[0];
  }
  da_update_step(st + PS_DA, acc / n, target);
  if (window_end) da_restart(st + PS_DA);
  const float eps = da_step_size(st + PS_DA);
  st[PS_EPS] = eps;
  const int t = (int)st[PS_T];
  if (eps_hist) eps_hist[t] = eps;
  st[PS_T] = (float)(t + 1);
  return n;
}

}  // namespace bjx
