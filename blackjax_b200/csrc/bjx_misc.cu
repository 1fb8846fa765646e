// Small kernels around the hot path: PRNG entry points (KAT-able), metric preparation,
// dual averaging / Welford window adaptation, chain-pooled summary statistics.
#include "bjx_internal.h"
#include "bjx_prng.cuh"
#include "bjx_da.cuh"

namespace bjx {

// ---- jax.random entry points --------------------------------------------------------------------------
__global__ void k_prng_split(const uint32_t* __restrict__ keys, long long n_keys, int num, uint32_t* __restrict__ out) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_keys * num) return;
  const long long k = t / num;
  const Key o = fold_in(Key{keys[2 * k], keys[2 * k + 1]}, (uint32_t)(t % num));
  out[2 * t] = o.a;
  out[2 * t + 1] = o.b;
}
__global__ void k_prng_fold_in(const uint32_t* __restrict__ keys, long long n_keys, uint32_t data, uint32_t* __restrict__ out) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_keys) return;
  const Key o = fold_in(Key{keys[2 * t], keys[2 * t + 1]}, data);
  out[2 * t] = o.a;
  out[2 * t + 1] = o.b;
}
template <int MODE>  // 0 bits, 1 uniform, 2 normal
__global__ void k_prng_draw(const uint32_t* __restrict__ keys, long long n_keys, long long per_key, void* __restrict__ out) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_keys * per_key) return;
  const long long k = t / per_key;
  const uint32_t i = (uint32_t)(t % per_key);
  const Key key{keys[2 * k], keys[2 * k + 1]};
  if (MODE == 0) reinterpret_cast<uint32_t*>(out)[t] = random_bits(key, i);
  if (MODE == 1) reinterpret_cast<float*>(out)[t] = bits_to_unit(random_bits(key, i));
  if (MODE == 2) reinterpret_cast<float*>(out)[t] = normal_at(key, i);
}

// jax.random.randint for int32 (randint_at, bjx_prng.cuh)
__global__ void k_prng_randint(const uint32_t* __restrict__ keys, long long n_keys, long long per_key, int minval,
                               int maxval, int* __restrict__ out) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_keys * per_key) return;
  const long long k = t / per_key;
  const Key key{keys[2 * k], keys[2 * k + 1]};
  out[t] = randint_at(key, (uint32_t)(t % per_key), minval, maxval);
}

static inline dim3 grid1d(long long n, int b = 256) { return dim3((unsigned)((n + b - 1) / b)); }

void launch_prng_split(const uint32_t* keys, long long n, int num, uint32_t* out, cudaStream_t s) {
  if (n * num > 0) k_prng_split<<<grid1d(n * num), 256, 0, s>>>(keys, n, num, out);
}
void launch_prng_fold_in(const uint32_t* keys, long long n, uint32_t data, uint32_t* out, cudaStream_t s) {
  if (n > 0) k_prng_fold_in<<<grid1d(n), 256, 0, s>>>(keys, n, data, out);
}
void launch_prng_randint(const uint32_t* keys, long long n, long long per_key, int minval, int maxval, int* out,
                         cudaStream_t s) {
  if (n * per_key > 0) k_prng_randint<<<grid1d(n * per_key), 256, 0, s>>>(keys, n, per_key, minval, maxval, out);
}
void launch_prng_draw(int mode, const uint32_t* keys, long long n, long long per_key, void* out, cudaStream_t s) {
  if (n * per_key <= 0) return;
  if (mode == 0) k_prng_draw<0><<<grid1d(n * per_key), 256, 0, s>>>(keys, n, per_key, out);
  if (mode == 1) k_prng_draw<1><<<grid1d(n * per_key), 256, 0, s>>>(keys, n, per_key, out);
  if (mode == 2) k_prng_draw<2><<<grid1d(n * per_key), 256, 0, s>>>(keys, n, per_key, out);
}

// ---- metrics._format_covariance, diagonal branch (metrics.py:703-708): mass_matrix_sqrt = 1/sqrt(M^-1) ----
__global__ void k_diag_mass_sqrt(const float* __restrict__ imm, long long n, float* __restrict__ out) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n) out[t] = 1.0f / sqrtf(imm[t]);
}
void launch_diag_mass_sqrt(const float* imm, long long n, float* out, cudaStream_t s) {
  if (n > 0) k_diag_mass_sqrt<<<grid1d(n), 256, 0, s>>>(imm, n, out);
}

// ---- dual averaging (bjx_da.cuh), one state per chain: state [C,5] ---------------------------------------
__global__ void k_da_init(int C, float* __restrict__ st, const float* __restrict__ eps0, float* __restrict__ eps_out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  da_init(st + 5 * c, eps0[c]);
  if (eps_out) eps_out[c] = da_step_size(st + 5 * c);
}
__global__ void k_da_update(int C, float* __restrict__ st, const float* __restrict__ acc, float target,
                            float* __restrict__ eps_out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  da_update_step(st + 5 * c, acc[c], target);
  if (eps_out) eps_out[c] = da_step_size(st + 5 * c);
}
__global__ void k_da_reset(int C, float* __restrict__ st, float* __restrict__ eps_out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  da_restart(st + 5 * c);
  if (eps_out) eps_out[c] = da_step_size(st + 5 * c);
}
__global__ void k_da_final(int C, const float* __restrict__ st, float* __restrict__ eps_out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) eps_out[c] = da_final(st + 5 * c);
}
void launch_da(int op, int C, float* st, const float* in, float target, float* eps_out, cudaStream_t s) {
  if (C <= 0) return;
  if (op == 0) k_da_init<<<grid1d(C), 256, 0, s>>>(C, st, in, eps_out);
  if (op == 1) k_da_update<<<grid1d(C), 256, 0, s>>>(C, st, in, target, eps_out);
  if (op == 2) k_da_reset<<<grid1d(C), 256, 0, s>>>(C, st, eps_out);
  if (op == 3) k_da_final<<<grid1d(C), 256, 0, s>>>(C, st, eps_out);
}

// ---- Welford, diagonal, one accumulator per chain (adaptation/mass_matrix.py:411-442) ----------------------
__global__ void k_welford_update(long long n, const float* __restrict__ x, float* __restrict__ mean,
                                 float* __restrict__ m2, float count) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const float v = x[t];
  const float m = mean[t];
  const float delta = v - m;
  const float nm = m + delta / count;
  mean[t] = nm;
  m2[t] = m2[t] + delta * (v - nm);
}
// regularised inverse mass matrix (mass_matrix.py:335-357) and accumulator reset
__global__ void k_welford_final(long long n, float* __restrict__ mean, float* __restrict__ m2, float count,
                                float* __restrict__ imm) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const float cov = m2[t] / (count - 1.f);
  const float denom = count + 5.f;
  imm[t] = count / denom * cov + 5.f / denom * 1e-3f;
  mean[t] = 0.f;
  m2[t] = 0.f;
}
void launch_welford_update(long long n, const float* x, float* mean, float* m2, int count, cudaStream_t s) {
  if (n > 0) k_welford_update<<<grid1d(n), 256, 0, s>>>(n, x, mean, m2, (float)count);
}
void launch_welford_final(long long n, float* mean, float* m2, int count, float* imm, cudaStream_t s) {
  if (n > 0) k_welford_final<<<grid1d(n), 256, 0, s>>>(n, mean, m2, (float)count, imm);
}

// ---- Welford, dense, one accumulator per chain (adaptation/mass_matrix.py:411-442 with is_diagonal_matrix=False: what
// jax.vmap(window_adaptation(..., is_mass_matrix_diagonal=False).run) carries per chain) ----------------------------------
// m2[c,i,j] += (x_i - mean_new_i) * (x_j - mean_old_j)   (jnp.outer(updated_delta, delta), :427-433); the mean is
// updated by a second launch so that every element of the outer product sees the OLD mean.
__global__ void k_welford_dense_m2(int C, int D, const float* __restrict__ x, const float* __restrict__ mean,
                                   float* __restrict__ m2, float count) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)C * D * D) return;
  const int j = (int)(t % D), i = (int)((t / D) % D);
  const long long c = t / ((long long)D * D);
  const float xi = x[c * D + i], mi = mean[c * D + i], xj = x[c * D + j], mj = mean[c * D + j];
  const float di = xi - mi;
  const float ui = xi - (mi + di / count);
  m2[t] = m2[t] + ui * (xj - mj);
}
__global__ void k_welford_mean(long long n, const float* __restrict__ x, float* __restrict__ mean, float count) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const float m = mean[t];
  mean[t] = m + (x[t] - m) / count;
}
// regularised dense inverse mass matrix (mass_matrix.py:335-357: the shrinkage target is 1e-3 * identity) and reset
__global__ void k_welford_dense_final(int C, int D, float* __restrict__ mean, float* __restrict__ m2, float count,
                                      float* __restrict__ imm) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)C * D * D) return;
  const int j = (int)(t % D), i = (int)((t / D) % D);
  const float cov = m2[t] / (count - 1.f);
  const float denom = count + 5.f;
  imm[t] = count / denom * cov + ((i == j) ? 5.f / denom * 1e-3f : 0.f);
  m2[t] = 0.f;
  if (j == 0) mean[(t / ((long long)D * D)) * D + i] = 0.f;
}
void launch_welford_dense_update(int C, int D, const float* x, float* mean, float* m2, int count, cudaStream_t s) {
  const long long n = (long long)C * D * D;
  if (n <= 0) return;
  k_welford_dense_m2<<<grid1d(n), 256, 0, s>>>(C, D, x, mean, m2, (float)count);
  k_welford_mean<<<grid1d((long long)C * D), 256, 0, s>>>((long long)C * D, x, mean, (float)count);
}
void launch_welford_dense_final(int C, int D, float* mean, float* m2, int count, float* imm, cudaStream_t s) {
  const long long n = (long long)C * D * D;
  if (n > 0) k_welford_dense_final<<<grid1d(n), 256, 0, s>>>(C, D, mean, m2, (float)count, imm);
}

// mass_matrix_sqrt of one dense inverse mass matrix PER CHAIN (metrics.py:712-715: L = chol(M^-1) lower,
// mass_matrix_sqrt = solve_triangular(L, I, lower, trans) = L^-T), float64 like the shared dense metric's host
// factorisation.  One CTA per chain, D <= 64: L (strict lower triangle) and L^-1 (stored transposed in the strict upper
// triangle) share one D x D shared-memory matrix, the two diagonals sit beside it.  A matrix that is not positive
// definite yields NaNs (as jnp.linalg.cholesky does).
__global__ void __launch_bounds__(64) k_chol_linv_t(int D, const float* __restrict__ imm, float* __restrict__ msqrt) {
  extern __shared__ double chol_sm[];
  double* S = chol_sm;            // [D, D]
  double* dL = chol_sm + D * D;   // diag(L)
  double* dI = dL + D;            // diag(L^-1)
  const int t = threadIdx.x;
  const float* A = imm + (size_t)blockIdx.x * D * D;
  float* out = msqrt + (size_t)blockIdx.x * D * D;
  for (int j = 0; j < D; ++j) {   // column j of L (Cholesky-Crout): thread t owns row t
    if (t == j) {
      double s = (double)A[(size_t)j * D + j];
      for (int k = 0; k < j; ++k) s -= S[j * D + k] * S[j * D + k];
      dL[j] = sqrt(s);
    }
    __syncthreads();
    if (t > j && t < D) {
      double s = (double)A[(size_t)t * D + j];
      for (int k = 0; k < j; ++k) s -= S[t * D + k] * S[j * D + k];
      S[t * D + j] = s / dL[j];
    }
    __syncthreads();
  }
  if (t < D) {                    // column t of L^-1 by forward substitution (thread-private column, stored at S[t][i])
    dI[t] = 1.0 / dL[t];
    for (int i = t + 1; i < D; ++i) {
      double s = -S[i * D + t] * dI[t];
      for (int k = t + 1; k < i; ++k) s -= S[i * D + k] * S[t * D + k];
      S[t * D + i] = s / dL[i];
    }
  }
  __syncthreads();
  // msqrt = (L^-1)^T: msqrt[i][j] = Linv[j][i] = (j > i ? S[i][j] : j == i ? dI[i] : 0)
  for (int e = t; e < D * D; e += blockDim.x) {
    const int i = e / D, j = e % D;
    out[e] = (float)(j > i ? S[i * D + j] : (j == i ? dI[i] : 0.0));
  }
}
void launch_chol_linv_t(int C, int D, const float* imm, float* msqrt, cudaStream_t s) {
  if (C <= 0) return;
  const size_t smem = ((size_t)D * D + 2 * D) * sizeof(double);
  k_chol_linv_t<<<C, 64, smem, s>>>(D, imm, msqrt);
}

// ---- chain-pooled summary block (metric_buffers.py:396-420 cgl_update_batch statistics) -------------------
// out[0] = sum acceptance_rate, out[1] = C, out[2:2+D] = mean over chains, out[2+D:2+2D] = sum (x-mean)^2.
// Column reductions over the chain axis: block (32 x 8) owns 32 columns, threads stride over chains
// (coalesced 128-byte rows), deterministic shared-memory tree, two passes (mean, then centred M2).
__global__ void k_pooled_colstats(int C, int D, const float* __restrict__ x, float* __restrict__ out) {
  __shared__ float red[8][33];
  const int col = blockIdx.x * 32 + threadIdx.x;
  float acc = 0.f;
  if (col < D)
    for (int c = threadIdx.y; c < C; c += 8) acc += x[(size_t)c * D + col];
  red[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  float mean = 0.f;
  if (threadIdx.y == 0) {
    float s = 0.f;
    for (int k = 0; k < 8; ++k) s += red[k][threadIdx.x];
    red[0][threadIdx.x] = s / (float)C;
  }
  __syncthreads();
  mean = red[0][threadIdx.x];
  __syncthreads();
  acc = 0.f;
  if (col < D)
    for (int c = threadIdx.y; c < C; c += 8) {
      const float d = x[(size_t)c * D + col] - mean;
      acc = fmaf(d, d, acc);
    }
  red[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && col < D) {
    float s = 0.f;
    for (int k = 0; k < 8; ++k) s += red[k][threadIdx.x];
    out[2 + col] = mean;
    out[2 + D + col] = s;
  }
}
__global__ void k_pooled_accept(int C, const float* __restrict__ acc, float* __restrict__ out) {
  __shared__ float red[32];
  float a = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) a += acc[c];
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = a;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int k = 0; k < (int)(blockDim.x >> 5); ++k) s += red[k];
    out[0] = s;
    out[1] = (float)C;
  }
}
// Dense pooled second moment: M2[i,j] = sum_c (x_ci - mean_i)(x_cj - mean_j)  (metric_buffers.py:396-420, dense
// branch `centered.T @ centered`).  Two deterministic stages: Z chain slices -> partial [Z, D, D], then the sum.
constexpr int kM2Slices = 32;
__global__ void k_pooled_m2_partial(int C, int D, const float* __restrict__ x, const float* __restrict__ mean,
                                    float* __restrict__ partial) {
  __shared__ float xi[32][17], xj[32][17];
  const int ti = threadIdx.x & 15, tj = threadIdx.x >> 4;
  const int i0 = blockIdx.x * 16, j0 = blockIdx.y * 16, z = blockIdx.z;
  const int per = (C + kM2Slices - 1) / kM2Slices;
  const int c0 = z * per, c1 = min(C, c0 + per);
  float acc = 0.f;
  for (int cb = c0; cb < c1; cb += 32) {
    for (int t = threadIdx.x; t < 32 * 16; t += 256) {
      const int cc = cb + t / 16, k = t % 16;
      const bool ok = cc < c1;
      xi[t / 16][k] = (ok && i0 + k < D) ? x[(size_t)cc * D + i0 + k] - mean[i0 + k] : 0.f;
      xj[t / 16][k] = (ok && j0 + k < D) ? x[(size_t)cc * D + j0 + k] - mean[j0 + k] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 32; ++r) acc = fmaf(xi[r][ti], xj[r][tj], acc);
    __syncthreads();
  }
  if (i0 + ti < D && j0 + tj < D) partial[((size_t)z * D + i0 + ti) * D + j0 + tj] = acc;
}
__global__ void k_pooled_m2_sum(int D, const float* __restrict__ partial, float* __restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= D * D) return;
  float s = 0.f;
  for (int z = 0; z < kM2Slices; ++z) s += partial[(size_t)z * D * D + t];
  out[t] = s;
}
__global__ void k_copy_f32(int n, const float* __restrict__ src, float* __restrict__ dst) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n) dst[t] = src[t];
}
// out = (sum acc, C, mean[D], M2[D,D]); scratch >= kM2Slices*D*D floats
void launch_pooled_stats_dense(int C, int D, const float* x, const float* acc, float* out, float* scratch, cudaStream_t s) {
  k_pooled_accept<<<1, 1024, 0, s>>>(C, acc, out);
  k_pooled_colstats<<<dim3((D + 31) / 32), dim3(32, 8), 0, s>>>(C, D, x, scratch);  // scratch[2:2+D] = mean (diag M2 unused)
  float* partial = scratch + 2 + 2 * (size_t)D;
  k_pooled_m2_partial<<<dim3((D + 15) / 16, (D + 15) / 16, kM2Slices), 256, 0, s>>>(C, D, x, scratch + 2, partial);
  k_copy_f32<<<(D + 255) / 256, 256, 0, s>>>(D, scratch + 2, out + 2);
  k_pooled_m2_sum<<<(D * D + 255) / 256, 256, 0, s>>>(D, partial, out + 2 + D);
}
size_t pooled_dense_scratch_floats(int D) { return 2 + 2 * (size_t)D + (size_t)kM2Slices * D * D; }

// ---- potential scale reduction (blackjax/diagnostics.py:39-89) over a device-resident history [T, C, D] ---------
// stage 1: per (chain, dim) sample mean and unbiased variance over the T draws (coalesced along D);
// stage 2 (k_pooled_colstats twice): across-chain mean / sum of squared deviations of those two [C,D] arrays.
__global__ void k_chain_moments(int T, long long CD, const float* __restrict__ hist, float* __restrict__ mean,
                                float* __restrict__ var) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= CD) return;
  float m = 0.f, m2 = 0.f;
  for (int i = 0; i < T; ++i) {  // Welford over the draws
    const float x = __ldcs(hist + (size_t)i * CD + t);
    const float d = x - m;
    m += d / (float)(i + 1);
    m2 = fmaf(d, x - m, m2);
  }
  mean[t] = m;
  var[t] = m2 / (float)(T - 1);
}
__global__ void k_rhat_finish(int T, int C, int D, const float* __restrict__ stats_mean, const float* __restrict__ stats_var,
                              float* __restrict__ rhat) {
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= D) return;
  // stats_* = (unused, C, mean over chains [D], sum sq. dev. over chains [D]) as written by k_pooled_colstats
  const float between = (float)T * (stats_mean[2 + D + d] / (float)(C - 1));  // num_samples * var(per-chain means, ddof=1)
  const float within = stats_var[2 + d];                                         // mean of the per-chain variances
  const float est = (float)(T - 1) / (float)T * within + between / (float)T;
  rhat[d] = sqrtf(est / within);
}
// scratch: 2*C*D + 2*(2+2D) floats
void launch_rhat(int T, int C, int D, const float* hist, float* rhat, float* scratch, cudaStream_t s) {
  float* mean = scratch;
  float* var = scratch + (size_t)C * D;
  float* st_m = var + (size_t)C * D;
  float* st_v = st_m + 2 + 2 * (size_t)D;
  k_chain_moments<<<grid1d((long long)C * D), 256, 0, s>>>(T, (long long)C * D, hist, mean, var);
  k_pooled_colstats<<<dim3((D + 31) / 32), dim3(32, 8), 0, s>>>(C, D, mean, st_m);
  k_pooled_colstats<<<dim3((D + 31) / 32), dim3(32, 8), 0, s>>>(C, D, var, st_v);
  k_rhat_finish<<<(D + 255) / 256, 256, 0, s>>>(T, C, D, st_m, st_v, rhat);
}

// ---- effective sample size (blackjax/diagnostics.py:159-305) over a device-resident history [T, C, D] -----------
// stage 1: per (chain, dim) sample mean (:210) and "differs from its first draw anywhere" flag (:203-208)
__global__ void k_ess_chain_mean(int T, int C, int D, const float* __restrict__ hist, float* __restrict__ mean,
                                 int* __restrict__ has_var) {
  const long long CD = (long long)C * D;
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= CD) return;
  const float x0 = hist[t];
  double acc = 0.0;
  bool varies = false;
  for (int i = 0; i < T; ++i) {
    const float x = __ldcs(hist + (size_t)i * CD + t);
    acc += (double)x;
    varies |= (x != x0);
  }
  mean[t] = (float)(acc / (double)T);
  if (varies) atomicOr(has_var + (int)(t % D), 1);
}

// stage 2: acov[lag, d] += sum over chains and draws of (x[s] - m)(x[s + lag] - m)  -- the zero-padded (linear)
// autocovariance the reference gets from its FFT (:212-221), evaluated directly.  A thread owns one (chain, dim) series
// (32 consecutive dims per warp: coalesced), a block of 8 warps walks a chunk of chains, blockIdx.y picks a block of 32
// lags; per 8 draws x 32 lags the inner product is 256 FMAs on 16 newly loaded values, all in registers.
constexpr int kEssLags = 32;
constexpr int kEssDraws = 8;
constexpr int kEssWarps = 8;
__global__ void __launch_bounds__(kEssWarps * 32) k_ess_autocov(int T, int C, int D, const float* __restrict__ hist,
                                                               const float* __restrict__ mean, double* __restrict__ acov,
                                                               int chains_per_block) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int d = blockIdx.x * 32 + lane;
  const int lag0 = blockIdx.y * kEssLags;
  const bool live = d < D;
  const size_t CD = (size_t)C * D;
  float acc[kEssLags];
#pragma unroll
  for (int l = 0; l < kEssLags; ++l) acc[l] = 0.f;
  const int c_end = min(C, (int)(blockIdx.z + 1) * chains_per_block);
  for (int c = blockIdx.z * chains_per_block + warp; c < c_end; c += kEssWarps) {
    const float m = live ? mean[(size_t)c * D + d] : 0.f;
    const float* series = hist + (size_t)c * D + (live ? d : 0);
    auto at = [&](int s) -> float { return (live && s < T) ? series[(size_t)s * CD] - m : 0.f; };
    // window w[i] = x[s + lag0 + i], i < kEssLags + kEssDraws; a[i] = x[s + i], i < kEssDraws
    float a[kEssDraws], w[kEssLags + kEssDraws];
#pragma unroll
    for (int i = 0; i < kEssLags; ++i) w[i] = at(lag0 + i);
    for (int s = 0; s < T - lag0; s += kEssDraws) {
#pragma unroll
      for (int i = 0; i < kEssDraws; ++i) {
        a[i] = at(s + i);
        w[kEssLags + i] = at(s + lag0 + kEssLags + i);
      }
#pragma unroll
      for (int i = 0; i < kEssDraws; ++i) {
#pragma unroll
        for (int l = 0; l < kEssLags; ++l) acc[l] = fmaf(a[i], w[i + l], acc[l]);
      }
#pragma unroll
      for (int i = 0; i < kEssLags; ++i) w[i] = w[i + kEssDraws];
    }
  }
  __shared__ float red[kEssWarps][kEssLags][32];
#pragma unroll
  for (int l = 0; l < kEssLags; ++l) red[warp][l][lane] = acc[l];
  __syncthreads();
  for (int l = warp; l < kEssLags; l += kEssWarps) {
    float sum = 0.f;
#pragma unroll
    for (int w = 0; w < kEssWarps; ++w) sum += red[w][l][lane];
    if (live && lag0 + l < T) atomicAdd(acov + (size_t)(lag0 + l) * D + d, (double)sum);
  }
}

// stage 3, one thread per dim: Geyer's initial positive / initial monotone sequences on the chain-averaged
// autocorrelation (:222-301).  The reference builds arrays with scans and a scatter; here the pairs are regenerated on
// the fly.  Its index max_t + 1 can be one past the last pair: JAX drops that scatter and clamps that gather.
__global__ void k_ess_finish(int T, int C, int D, const float* __restrict__ mean, const int* __restrict__ has_var,
                             const double* __restrict__ acov, float* __restrict__ ess) {
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= D) return;
  const double norm = 1.0 / ((double)T * (double)C);
  auto a = [&](int t) -> float { return (float)(acov[(size_t)t * D + d] * norm); };
  const float Tf = (float)T;
  const float var0 = a(0) * Tf / (Tf - 1.0f);                                      // :222-226
  const bool degenerate = isfinite(var0) && (!has_var[d] || var0 <= 0.0f);         // :227-229
  float wvar = var0 * (Tf - 1.0f) / Tf;                                            // :230
  if (C > 1) {                                                                     // :231-237 var of the chain means, ddof=1
    double s1 = 0.0, s2 = 0.0;
    for (int c = 0; c < C; ++c) {
      const double v = (double)mean[(size_t)c * D + d];
      s1 += v;
      s2 += v * v;
    }
    wvar += (float)((s2 - s1 * s1 / (double)C) / (double)(C - 1));
  }
  if (degenerate) wvar = 1.0f;                                                     // :238-240
  const int K = (T - T % 2) / 2;                                                   // pairs (rho[2k], rho[2k+1])
  auto rho = [&](int t) -> float { return t == 0 ? 1.0f : 1.0f - (var0 - a(t)) / wvar; };   // :243-253
  int n_true = 0;                                                                  // :259-270 leading run of positive pairs
  while (n_true < K && rho(2 * n_true) + rho(2 * n_true + 1) > 0.0f) ++n_true;
  const int max_t = n_true > 0 ? n_true - 1 : 0;
  const int idx = max_t + 1, idx_get = idx < K ? idx : K - 1;
  const bool even_at_idx = rho(2 * idx_get) > 0.0f;                                // :273 (unmasked value)
  float carry = 0.f, sum = 0.f, e_at = 0.f;
  const int k_end = (idx + 1 < K) ? idx + 1 : K;                                   // every later pair is masked to zero
  for (int k = 0; k < k_end; ++k) {
    const bool mk = k < n_true;
    const bool mk_even = (k == idx) ? even_at_idx : mk;                            // :273
    float e = mk_even ? rho(2 * k) : 0.f;                                          // :274
    float o = mk ? rho(2 * k + 1) : 0.f;                                           // :271
    const float s = e + o;
    if (k == 0) carry = s;                                                         // :282-285
    const bool upd = s > carry;                                                    // :277-280
    const float nxt = upd ? carry : s;
    carry = nxt;
    if (upd) e = o = nxt / 2.0f;                                                   // :287-288
    sum += e + o;
    if (k == idx_get) e_at = e;
  }
  const float ess_raw = (float)C * (float)T;                                       // :292
  float tau = -1.0f + 2.0f * sum - e_at;                                           // :293-297
  tau = fmaxf(tau, 1.0f / log10f(ess_raw));                                        // :299
  ess[d] = degenerate ? 0.0f : ess_raw / tau;                                      // :300-301
}

size_t ess_scratch_floats(int T, int C, int D) { return 2 * (size_t)T * D + (size_t)C * D + (size_t)D + 8; }
// scratch (8-byte aligned): acov double [T, D] | mean float [C, D] | has_var int [D]
void launch_ess(int T, int C, int D, const float* hist, float* ess, float* scratch, cudaStream_t s) {
  double* acov = reinterpret_cast<double*>(scratch);
  float* mean = scratch + 2 * (size_t)T * D;
  int* has_var = reinterpret_cast<int*>(mean + (size_t)C * D);
  cudaMemsetAsync(acov, 0, sizeof(double) * (size_t)T * D, s);
  cudaMemsetAsync(has_var, 0, sizeof(int) * (size_t)D, s);
  k_ess_chain_mean<<<grid1d((long long)C * D), 256, 0, s>>>(T, C, D, hist, mean, has_var);
  const int lag_blocks = (T + kEssLags - 1) / kEssLags;
  // enough chain chunks to fill the GPU, few enough that the double atomics stay rare
  const int d_blocks = (D + 31) / 32;
  int chunks = (4 * sm_count() + d_blocks * lag_blocks - 1) / (d_blocks * lag_blocks);
  chunks = chunks < 1 ? 1 : chunks;
  const int max_chunks = (C + kEssWarps - 1) / kEssWarps;
  chunks = chunks > max_chunks ? max_chunks : chunks;
  const int cpb = (C + chunks - 1) / chunks;
  k_ess_autocov<<<dim3(d_blocks, lag_blocks, (C + cpb - 1) / cpb), kEssWarps * 32, 0, s>>>(T, C, D, hist, mean, acov, cpb);
  k_ess_finish<<<(D + 127) / 128, 128, 0, s>>>(T, C, D, mean, has_var, acov, ess);
}

// ---- single-chain ESS of every (chain, dim) series of a history [T, C, D] -----------------------------------------------
// effective_sample_size(history[:, c, None, :]) for every chain c (mclmc_adaptation.py:393): the arithmetic of k_ess_chain_mean,
// k_ess_autocov and k_ess_finish with C = 1, but a thread owns one series from its mean to its ESS.  Geyer's procedure reads
// the autocorrelation only up to the pair after the initial positive sequence, so the warp (32 dims of one chain) evaluates
// blocks of kEssLags lags, feeding each pair into the sequence as it arrives, until every series of the warp has ended its
// initial positive sequence and seen that next pair.  Each lag's sum is the same fmaf chain as k_ess_autocov's, and the
// pairs go through the same operations in the same order as k_ess_finish, so the result is that of evaluating all lags.
// lags_out (optional, zeroed by the caller): per chain, the most lags any of its warps evaluated.
__global__ void __launch_bounds__(128) k_ess_chain(int T, int C, int D, const float* __restrict__ hist, float* __restrict__ ess,
                                                   int* __restrict__ lags_out) {
  const int lane = threadIdx.x & 31;
  const int d_blocks = (D + 31) / 32;
  const long long w = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (w >= (long long)C * d_blocks) return;
  const int c = (int)(w / d_blocks);
  const int d = (int)(w % d_blocks) * 32 + lane;
  const bool live = d < D;
  const size_t CD = (size_t)C * D;
  const float* series = hist + (size_t)c * D + (live ? d : 0);
  // k_ess_chain_mean
  float m = 0.f;
  bool varies = false;
  if (live) {
    const float x0 = series[0];
    double acc = 0.0;
    for (int i = 0; i < T; ++i) {
      const float x = series[(size_t)i * CD];
      acc += (double)x;
      varies |= (x != x0);
    }
    m = (float)(acc / (double)T);
  }
  auto at = [&](int s) -> float { return (live && s < T) ? series[(size_t)s * CD] - m : 0.f; };
  const double norm = 1.0 / ((double)T * 1.0);
  const float Tf = (float)T;
  const int K = (T - T % 2) / 2;
  float var0 = 0.f, wvar = 1.f, carry = 0.f, sum = 0.f, e_at = 0.f;
  bool degenerate = false, done = !live;
  int lag0 = 0;
  for (;; lag0 += kEssLags) {
    // k_ess_autocov for lags lag0 .. lag0 + kEssLags - 1
    float acc[kEssLags];
#pragma unroll
    for (int l = 0; l < kEssLags; ++l) acc[l] = 0.f;
    float a[kEssDraws], win[kEssLags + kEssDraws];
#pragma unroll
    for (int i = 0; i < kEssLags; ++i) win[i] = at(lag0 + i);
    for (int s = 0; s < T - lag0; s += kEssDraws) {
#pragma unroll
      for (int i = 0; i < kEssDraws; ++i) {
        a[i] = at(s + i);
        win[kEssLags + i] = at(s + lag0 + kEssLags + i);
      }
#pragma unroll
      for (int i = 0; i < kEssDraws; ++i) {
#pragma unroll
        for (int l = 0; l < kEssLags; ++l) acc[l] = fmaf(a[i], win[i + l], acc[l]);
      }
#pragma unroll
      for (int i = 0; i < kEssLags; ++i) win[i] = win[i + kEssDraws];
    }
    if (lag0 == 0) {  // k_ess_finish :222-240 with C = 1
      var0 = (float)((double)acc[0] * norm) * Tf / (Tf - 1.0f);
      degenerate = isfinite(var0) && (!varies || var0 <= 0.0f);
      wvar = var0 * (Tf - 1.0f) / Tf;
      if (degenerate) wvar = 1.0f;
    }
    // pairs lag0 / 2 .. lag0 / 2 + kEssLags / 2 - 1 through Geyer's initial positive and monotone sequences (:243-297)
#pragma unroll
    for (int p = 0; p < kEssLags / 2; ++p) {
      const int k = lag0 / 2 + p;
      if (!done && k < K) {
        const float re = (k == 0) ? 1.0f : 1.0f - (var0 - (float)((double)acc[2 * p] * norm)) / wvar;
        const float ro = 1.0f - (var0 - (float)((double)acc[2 * p + 1] * norm)) / wvar;
        const bool positive = re + ro > 0.0f;
        if (!positive && k == 0) {  // no positive pair: every pair is masked to zero
          done = true;
        } else {
          // in the sequence: (re, ro); the pair after it (k == max_t + 1): its even term when positive, no odd term
          float e = positive ? re : (re > 0.0f ? re : 0.f);
          float o = positive ? ro : 0.f;
          const float sp = e + o;
          if (k == 0) carry = sp;
          const bool upd = sp > carry;
          const float nxt = upd ? carry : sp;
          carry = nxt;
          if (upd) e = o = nxt / 2.0f;
          sum += e + o;
          e_at = e;  // idx_get is the pair after the sequence, or the last pair when every pair is positive
          done = !positive;
        }
      }
    }
    if (lag0 + kEssLags >= 2 * K) done = true;  // every pair seen
    if (__all_sync(0xffffffffu, done)) break;
  }
  if (lags_out && lane == 0) atomicMax(lags_out + c, min(lag0 + kEssLags, T));
  if (!live) return;
  const float ess_raw = 1.0f * (float)T;                                           // :292
  float tau = -1.0f + 2.0f * sum - e_at;                                           // :293-297
  tau = fmaxf(tau, 1.0f / log10f(ess_raw));                                        // :299
  ess[(size_t)c * D + d] = degenerate ? 0.0f : ess_raw / tau;                      // :300-301
}

void launch_ess_per_chain(int T, int C, int D, const float* hist, float* ess, int* lags_out, cudaStream_t s) {
  const long long warps = (long long)C * ((D + 31) / 32);
  k_ess_chain<<<(unsigned)((warps + 3) / 4), 128, 0, s>>>(T, C, D, hist, ess, lags_out);
}

void launch_pooled_stats(int C, int D, const float* x, const float* acc, float* out, cudaStream_t s) {
  k_pooled_accept<<<1, 1024, 0, s>>>(C, acc, out);
  k_pooled_colstats<<<dim3((D + 31) / 32), dim3(32, 8), 0, s>>>(C, D, x, out);
}

}  // namespace bjx
