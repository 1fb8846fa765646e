// Internal declarations shared by the translation units of libbjx.so.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace bjx {
// SMs of the current device: sizes the fixed grids of the grid-stride kernels
inline int sm_count() {
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms > 0 ? sms : 1;
}
void launch_prng_split(const uint32_t* keys, long long n, int num, uint32_t* out, cudaStream_t s);
void launch_prng_fold_in(const uint32_t* keys, long long n, uint32_t data, uint32_t* out, cudaStream_t s);
void launch_prng_draw(int mode, const uint32_t* keys, long long n, long long per_key, void* out, cudaStream_t s);
void launch_diag_mass_sqrt(const float* imm, long long n, float* out, cudaStream_t s);
void launch_da(int op, int C, float* st, const float* in, float target, float* eps_out, cudaStream_t s);
void launch_welford_update(long long n, const float* x, float* mean, float* m2, int count, cudaStream_t s);
void launch_welford_final(long long n, float* mean, float* m2, int count, float* imm, cudaStream_t s);
void launch_welford_dense_update(int C, int D, const float* x, float* mean, float* m2, int count, cudaStream_t s);
void launch_welford_dense_final(int C, int D, float* mean, float* m2, int count, float* imm, cudaStream_t s);
void launch_chol_linv_t(int C, int D, const float* imm, float* msqrt, cudaStream_t s);
void launch_pooled_stats(int C, int D, const float* x, const float* acc, float* out, cudaStream_t s);
void launch_pooled_stats_dense(int C, int D, const float* x, const float* acc, float* out, float* scratch, cudaStream_t s);
size_t pooled_dense_scratch_floats(int D);
void launch_rhat(int T, int C, int D, const float* hist, float* rhat, float* scratch, cudaStream_t s);
void launch_prng_randint(const uint32_t* keys, long long n, long long per_key, int minval, int maxval, int* out,
                         cudaStream_t s);
size_t ess_scratch_floats(int T, int C, int D);
void launch_ess(int T, int C, int D, const float* hist, float* ess, float* scratch, cudaStream_t s);
// windowed D x D covariance accumulators of bjx_adapt.cu: cov_stat_blocks(C) blocks of cov_block_floats(D) floats (count,
// -, mean[D], m2[D, D] lower triangle); the fold uses nb * (2 + 2D) floats of stats scratch; the merge writes the full
// covariance m2 / max(n - 1, 1) [D, D] to out and (n, mean[D]) to count_mean
int cov_stat_blocks(int C);
size_t cov_block_floats(int D);
void launch_cov_fold(int C, int D, const float* q, float* stats, float* cov, cudaStream_t s);
void launch_cov_merge(int C, int D, const float* cov, float* out, float* count_mean, cudaStream_t s);
}  // namespace bjx
