// Internal declarations shared by the translation units of libbjx.so.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

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
// per-chain dual averaging on st [C, 5] (bjx_da.cuh): op 0 init from in = eps0 [C], 1 update on in = acceptance [C], 2 restart,
// 3 final; eps_out [C] (optional for 0-2) takes the step size
void launch_da(int op, int C, float* st, const float* in, float target, float* eps_out, cudaStream_t s);
// dst[i] = src[0], i < n: a device scalar broadcast to the per-chain array the transition kernels read
void launch_fill_from(int n, const float* src, float* dst, cudaStream_t s);
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
// single-chain ESS of every (chain, dim) series: ess [C, D]; lags_out (optional, zeroed) [C] lags evaluated per chain
void launch_ess_per_chain(int T, int C, int D, const float* hist, float* ess, int* lags_out, cudaStream_t s);
// the tuners' per-chain key tree (bjx_mclmc_tune.cu): part1[c], part2[c] = split(k_c) with k_c the chain's key
// (split(keys[0:2], n_global)[chain_offset + c] when key_shared, else keys[c]); out[c] = split(base[c], n)[i]
void launch_tune_part_keys(int C, int key_shared, uint32_t chain_offset, const uint32_t* keys, uint32_t* part1,
                           uint32_t* part2, cudaStream_t s);
void launch_tune_fold_keys(int C, const uint32_t* base, uint32_t i, uint32_t* out, cudaStream_t s);
// windowed D x D covariance accumulators of bjx_adapt.cu: cov_stat_blocks(C) blocks of cov_block_floats(D) floats (count,
// -, mean[D], m2[D, D] lower triangle).  launch_block_stats writes the nb records (sum acc, n, mean[D], M2[D]) of the
// statistic blocks of x [C, D] to out; the fold takes these records of q as stats.  The merge of nblk accumulators writes
// the full covariance m2 / max(n - 1, 1) [D, D], whitened by imm unless it is null, to out and (n, mean[D]) to count_mean
// unless it is null.
int cov_stat_blocks(int C);
size_t cov_block_floats(int D);
void launch_block_stats(int C, int D, const float* x, const float* acc, float* out, cudaStream_t s);
void launch_cov_fold(int C, int D, const float* q, const float* stats, float* cov, cudaStream_t s);
void launch_cov_merge(int nblk, int D, const float* cov, const float* imm, float* out, float* count_mean, cudaStream_t s);
}  // namespace bjx

// Host-side routing and run-loop helpers of bjx_api.cu, shared with the entry points of other translation units.
typedef struct bjx_handle_s* bjx_handle_t;
namespace bjx {
struct Params;
struct LaunchArgs;
}  // namespace bjx
// Execution path of a call.  ROUTE_ROWS: the warp-per-chain row kernels (dim <= 1024, bjx_launch.cuh); ROUTE_BIG: the
// CTA-per-chain kernels (1024 < dim, bjx_big.cu); ROUTE_DENSE: the tensor-core dense path (bjx_dense.cu), taken by a dense
// Gaussian target or a dense metric beyond 128 dims.
enum Route { ROUTE_ROWS, ROUTE_BIG, ROUTE_DENSE };
Route transition_route(bjx_handle_t h);                  // where a transition, which needs target and metric, runs
Route target_route(bjx_handle_t h);                      // where a kernel that needs the target only runs
bjx::Params make_params(bjx_handle_t h, float eps, const float* eps_dev);
// launches kernel_id of the handle's (target, size class, metric, integrator) variant; target_dependent = false takes the
// target-independent instance
int dispatch(bjx_handle_t h, int kernel_id, bool target_dependent, bjx::LaunchArgs& a);
// null handle / metric not set / null or misaligned state arrays; selects the handle's device
int check_ready(bjx_handle_t h, bool need_metric, const void* const* ptrs, int n);
// split(rng_key, num_steps) into h->sample_keys (util.py:203)
int split_step_keys(bjx_handle_t h, const uint32_t* rng_key, int num_steps);
// L = chol(a) (lower, row-major [D, D]) in float64 from the float32 [D, D] a; false when a is not positive definite
bool cholesky_f64(const std::vector<float>& a, int D, std::vector<double>& L);
// bjx_mclmc.cu: dim >= 2, a diagonal metric and the row kernels, or BJX_E_UNSUPPORTED with "<name> ..." as the reason
int mclmc_transition_supported(bjx_handle_t h, const char* name);
// bjx_meads.cu, shared with the low-rank window adaptation (bjx_lowrank_window.cu): the install of (sigma, U, lam) into a
// rank-k low-rank metric block (k_lrd_install).
void launch_lrd_install(int D, int k, const float* sigma, const float* U, const float* lam, float* blk, cudaStream_t s);
