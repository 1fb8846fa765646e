// MEADS warm-up statistics for generalized HMC, the chain shuffle, device resident.
//
// Reference semantics (blackjax/adaptation/meads_adaptation.py:497-690, low_rank_rank=None): the chains are split into
// K contiguous folds; per warm-up step and fold k
//   scale_k    = std over the fold's chains of the positions                                   (:516)
//   eps_own_k  = min(multiplier / sqrt(max_eig(grad * scale_k)), 1)                            (:551-559)
//   eps_k, scale_k handed to fold k+1 (roll by one)                                             (:560-563)
//   gamma_k    = max(1 / sqrt(max_eig(position / scale_k - mean)), slowdown / ((t+1) eps_k))   (:565-572)
//   alpha_k    = 1 - exp(-2 eps_k gamma_k), delta_k = alpha_k / 2                              (:573-575)
// with max_eig(X) = [(sum(S^2) - sum(diag(S)^2)) / (n(n-1))] / [sum(diag(S)) / n], S = X X^T   (:805-817).
// The reference forms the n x n Gram matrix S; here sum(S^2) = ||X^T X||_F^2 is taken from the D x D Gram matrix in
// 32 x 32 tiles (upper triangle, off-diagonal tiles counted twice) -- D^2 n flops instead of n^2 D -- and diag(S) from
// one warp per chain.  Every reduction runs in a fixed order, so results are reproducible run to run.
// jax.random.permutation for the shuffle every K steps (:675-683) is JAX's sort-based shuffle (jax/_src/random.py
// _shuffle: ceil(3 ln n / ln(2^32-1)) rounds of a stable sort by 32 fresh random bits): a bitonic sort of the 64-bit
// composites (bits << 32 | position), which orders ties by position exactly like a stable sort.
#include <cooperative_groups.h>

#include <algorithm>
#include <cmath>
#include <mutex>

#include "bjx_handle.h"
#include "bjx_internal.h"
#include "bjx_lrd_eig.cuh"

namespace bjx {

// grid (ceil(D/32), K), block (32, 8): mean, population std and mean of position/std per (fold, dim)
__global__ void k_meads_moments(int n, int D, const float* __restrict__ q, float* __restrict__ mu, float* __restrict__ sd,
                                float* __restrict__ mus) {
  __shared__ float red[8][33];
  const int col = blockIdx.x * 32 + threadIdx.x;
  const size_t c0 = (size_t)blockIdx.y * n;
  auto reduce = [&](float a) {
    red[threadIdx.y][threadIdx.x] = a;
    __syncthreads();
    float s = 0.f;
    for (int k = 0; k < 8; ++k) s += red[k][threadIdx.x];
    __syncthreads();
    return s;
  };
  float a = 0.f;
  if (col < D)
    for (int c = threadIdx.y; c < n; c += 8) a += q[(c0 + c) * D + col];
  const float mean = reduce(a) / (float)n;
  a = 0.f;
  if (col < D)
    for (int c = threadIdx.y; c < n; c += 8) {
      const float d = q[(c0 + c) * D + col] - mean;
      a = fmaf(d, d, a);
    }
  const float s = sqrtf(reduce(a) / (float)n);  // jnp.std, ddof = 0
  a = 0.f;
  if (col < D)
    for (int c = threadIdx.y; c < n; c += 8) a += q[(c0 + c) * D + col] / s;
  const float ms = reduce(a) / (float)n;
  if (col < D && threadIdx.y == 0) {
    const size_t o = (size_t)blockIdx.y * D + col;
    mu[o] = mean;
    sd[o] = s;
    mus[o] = ms;
  }
}

__device__ __forceinline__ float meads_x(int which, float qv, float gv, float s, float ms) {
  return which == 0 ? gv * s : qv / s - ms;
}

// one warp per chain: diag(S) of both matrices
__global__ void k_meads_rows(int C, int n, int D, const float* __restrict__ q, const float* __restrict__ g,
                             const float* __restrict__ sd, const float* __restrict__ mus, float* __restrict__ rg,
                             float* __restrict__ rq) {
  const int chain = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (chain >= C) return;
  const size_t f = (size_t)(chain / n) * D;
  float a = 0.f, b = 0.f;
  for (int d = lane; d < D; d += 32) {
    const float s = sd[f + d];
    const float x = g[(size_t)chain * D + d] * s;
    const float y = q[(size_t)chain * D + d] / s - mus[f + d];
    a = fmaf(x, x, a);
    b = fmaf(y, y, b);
  }
  a = warp_sum(a);
  b = warp_sum(b);
  if (lane == 0) {
    rg[chain] = a;
    rq[chain] = b;
  }
}

// grid (pairs, 2, K), block (32, 32): one 32 x 32 tile of X^T X (upper triangle of tiles), reduced to its sum of squares
__global__ void __launch_bounds__(1024) k_meads_gram(int n, int D, int T, const float* __restrict__ q,
                                                     const float* __restrict__ g, const float* __restrict__ sd,
                                                     const float* __restrict__ mus, float* __restrict__ tiles) {
  __shared__ float As[32][33], Bs[32][33];
  __shared__ float wsum[32];
  int bi = 0, rem = blockIdx.x;
  while (rem >= T - bi) {
    rem -= T - bi;
    ++bi;
  }
  const int bj = bi + rem;
  const int which = blockIdx.y, fold = blockIdx.z;
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int da = bi * 32 + tx, db = bj * 32 + tx;
  const size_t f = (size_t)fold * D;
  const float sa = da < D ? sd[f + da] : 1.f, ma = da < D ? mus[f + da] : 0.f;
  const float sb = db < D ? sd[f + db] : 1.f, mb = db < D ? mus[f + db] : 0.f;
  const float* src = which == 0 ? g : q;
  float acc = 0.f;
  for (int c0 = 0; c0 < n; c0 += 32) {
    const int c = c0 + ty;
    float xa = 0.f, xb = 0.f;
    if (c < n) {
      const size_t row = ((size_t)fold * n + c) * D;
      if (da < D) xa = meads_x(which, src[row + da], src[row + da], sa, ma);
      if (db < D) xb = meads_x(which, src[row + db], src[row + db], sb, mb);
    }
    As[ty][tx] = xa;
    Bs[ty][tx] = xb;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 32; ++k) acc = fmaf(As[k][ty], Bs[k][tx], acc);
    __syncthreads();
  }
  float v = warp_sum(acc * acc);
  if (tx == 0) wsum[ty] = v;
  __syncthreads();
  if (ty == 0) {
    v = warp_sum(wsum[tx]);
    if (tx == 0) tiles[((size_t)fold * 2 + which) * gridDim.x + blockIdx.x] = (bi == bj) ? v : 2.f * v;
  }
}

// jnp.minimum / jnp.maximum propagate NaN (fminf / fmaxf drop it)
__device__ __forceinline__ float nan_min(float a, float b) { return (isnan(a) || isnan(b)) ? a + b : fminf(a, b); }
__device__ __forceinline__ float nan_max(float a, float b) { return (isnan(a) || isnan(b)) ? a + b : fmaxf(a, b); }

// one CTA: sums, max_eig, fold parameters, roll, metric rows
// state: step_size[K] | alpha[K] | delta[K] | sigma[K,D] | imm[K,D] | msqrt[K,D]
__global__ void k_meads_finish(int n, int D, int K, int pairs, int t, float multiplier, float slowdown,
                               const float* __restrict__ sd, const float* __restrict__ rg, const float* __restrict__ rq,
                               const float* __restrict__ tiles, float* __restrict__ state) {
  __shared__ double red[256];
  __shared__ float eig[64][2];
  __shared__ float own[64];
  auto block_sum = [&](double a) {
    red[threadIdx.x] = a;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
      if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
      __syncthreads();
    }
    const double s = red[0];
    __syncthreads();
    return s;
  };
  for (int k = 0; k < K; ++k)
    for (int which = 0; which < 2; ++which) {
      const float* r = (which == 0 ? rg : rq) + (size_t)k * n;
      double a = 0.0, b = 0.0, c = 0.0;
      for (int i = threadIdx.x; i < n; i += 256) {
        const double v = r[i];
        a += v;
        b += v * v;
      }
      const float* tl = tiles + ((size_t)k * 2 + which) * pairs;
      for (int i = threadIdx.x; i < pairs; i += 256) c += tl[i];
      const double sr = block_sum(a), sr2 = block_sum(b), s2 = block_sum(c);
      if (threadIdx.x == 0) {
        const float lam = (float)sr / (float)n;
        const float lam_sq = (float)(s2 - sr2) / (float)((double)n * (double)(n - 1));
        eig[k][which] = lam_sq / lam;
      }
    }
  __syncthreads();
  if ((int)threadIdx.x < K) own[threadIdx.x] = nan_min(multiplier / sqrtf(eig[threadIdx.x][0]), 1.0f);
  __syncthreads();
  if ((int)threadIdx.x < K) {
    const int k = threadIdx.x;
    const float eps = own[(k + K - 1) % K];
    const float gamma = nan_max(1.0f / sqrtf(eig[k][1]), slowdown / ((float)(t + 1) * eps));
    const float alpha = 1.0f - expf(-2.0f * eps * gamma);
    state[k] = eps;
    state[K + k] = alpha;
    state[2 * K + k] = alpha / 2.0f;
  }
  float* sig = state + 3 * K;
  float* imm = sig + (size_t)K * D;
  float* msq = imm + (size_t)K * D;
  for (int i = threadIdx.x; i < K * D; i += 256) {
    const int k = i / D, d = i - k * D;
    const float s = sd[(size_t)((k + K - 1) % K) * D + d];
    const float m = s * s;                      // ghmc.py:84: inverse scale squared
    sig[i] = s;
    imm[i] = m;
    msq[i] = 1.0f / sqrtf(m);                   // metrics.py:699-704
  }
}

// maximum_eigenvalue of one explicit matrix (which = 0 statistics with unit scales)
__global__ void k_fill2(float* __restrict__ a, int n, float va, float* __restrict__ b, float vb) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    a[i] = va;
    b[i] = vb;
  }
}
__global__ void k_maxeig_finish(int n, int pairs, const float* __restrict__ r, const float* __restrict__ tiles,
                                float* __restrict__ out) {
  __shared__ double red[256];
  auto block_sum = [&](double a) {
    red[threadIdx.x] = a;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
      if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
      __syncthreads();
    }
    const double s = red[0];
    __syncthreads();
    return s;
  };
  double a = 0.0, b = 0.0, c = 0.0;
  for (int i = threadIdx.x; i < n; i += 256) {
    const double v = r[i];
    a += v;
    b += v * v;
  }
  for (int i = threadIdx.x; i < pairs; i += 256) c += tiles[i];
  const double sr = block_sum(a), sr2 = block_sum(b), s2 = block_sum(c);
  if (threadIdx.x == 0) {
    const float lam = (float)sr / (float)n;
    const float lam_sq = (float)(s2 - sr2) / (float)((double)n * (double)(n - 1));
    out[0] = lam_sq / lam;
  }
}

// ---- jax.random.permutation --------------------------------------------------------------------------------------
__global__ void k_perm_keys(const uint32_t* __restrict__ key, long long fold_index, int round, int n, long long npow2,
                            unsigned long long* __restrict__ comp) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npow2) return;
  if (i >= n) {
    comp[i] = ~0ull;
    return;
  }
  Key k{key[0], key[1]};
  if (fold_index >= 0) k = fold_in(k, (uint32_t)fold_index);
  for (int r = 0; r < round; ++r) k = fold_in(k, 0u);  // key, subkey = split(key): key = child 0
  const Key sub = fold_in(k, 1u);
  comp[i] = ((unsigned long long)random_bits(sub, (uint32_t)i) << 32) | (unsigned long long)i;
}

__global__ void k_bitonic_step(unsigned long long* __restrict__ a, long long npow2, long long j, long long k) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npow2) return;
  const long long l = i ^ j;
  if (l <= i) return;
  const unsigned long long x = a[i], y = a[l];
  const bool up = (i & k) == 0;
  if ((x > y) == up) {
    a[i] = y;
    a[l] = x;
  }
}

__global__ void k_perm_apply(const unsigned long long* __restrict__ comp, const int* __restrict__ x_old, int* __restrict__ x_new,
                             int n) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int src = (int)(comp[j] & 0xffffffffull);
  x_new[j] = x_old ? x_old[src] : src;
}

__global__ void k_gather_rows(const int* __restrict__ perm, const float* __restrict__ src, float* __restrict__ dst, int rows,
                              int width) {
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= rows) return;
  const float* s = src + (size_t)perm[r] * width;
  float* d = dst + (size_t)r * width;
  for (int i = lane; i < width; i += 32) d[i] = s[i];
}

static int meads_pairs(int D) {
  const int T = (D + 31) / 32;
  return T * (T + 1) / 2;
}

// ---- MEADS-LRD (meads_adaptation.py:459-784 with low_rank_rank = k) -----------------------------------------------
// One low-rank metric (sigma, U, lam) for all chains per warm-up step.  In the window the positions of all chains are
// folded into the windowed covariance accumulators of bjx_adapt.cu (cgl_update_batch); once they hold 2 D samples the
// metric is the top-k eigenpairs by |lam - 1| of the pooled correlation matrix R (sample_covariance_eigh_low_rank,
// metric_estimators.py:543-615), else the diagonal fallback sigma = std of all positions, U = eye(D, k), lam = 1
// (:263-289).  lam is floored at 1e-6 (:292-313).
//


// lrd_state: header | sigma[D] U[D,k] lam[k] (this step's metric) | n, mean[D] of the merged accumulator | mu, sd, -
// [3D] of the final positions | Ritz basis [D, b] | merged covariance [D, D] | fold scratch | block accumulators
struct LrdLayout {
  size_t sigma, U, lam, cm, fin, basis, W, stats, cov, total;
};
static LrdLayout lrd_layout(int C, int D, int k) {
  LrdLayout L{};
  const size_t d = (size_t)D;
  const int nb = cov_stat_blocks(C);
  size_t o = kLrdHdr;
  L.sigma = o; o += d;
  L.U = o; o += d * k;
  L.lam = o; o += k;
  L.cm = o; o += 1 + d;
  L.fin = o; o += 3 * d;
  L.basis = o; o += d * lrd_basis_cols(D, k);
  L.W = o; o += d * d;
  L.stats = o; o += (size_t)nb * (2 + 2 * d);
  L.cov = o; o += (size_t)nb * cov_block_floats(D);
  L.total = o;
  return L;
}



// The gate and the diagonal fallback.  mu, sd [K, D]: mean and population std of each of K folds of n chains, pooled
// here into the std of all K n chains.  Writes the engagement flag; the metric only when not engaged.
__global__ void k_lrd_fallback(int D, int k, int K, int n, const float* __restrict__ mu, const float* __restrict__ sd,
                               int gate, const float* __restrict__ cm, float* __restrict__ hdr, float* __restrict__ sigma,
                               float* __restrict__ U, float* __restrict__ lam) {
  const bool engaged = gate && cm[0] >= 2.f * (float)D;
  if (threadIdx.x == 0) hdr[LRD_ENGAGED] = engaged ? 1.f : 0.f;
  if (engaged) return;
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float m = 0.f;
    for (int f = 0; f < K; ++f) m += mu[(size_t)f * D + d];
    m /= (float)K;
    float v = 0.f;
    for (int f = 0; f < K; ++f) {
      const float s = sd[(size_t)f * D + d], e = mu[(size_t)f * D + d] - m;
      v += s * s + e * e;
    }
    const float s = K == 1 ? sd[d] : sqrtf(v / (float)K);
    sigma[d] = s <= 0.f ? 1.f : s;
    for (int j = 0; j < k; ++j) U[(size_t)d * k + j] = d == j ? 1.f : 0.f;
  }
  for (int j = threadIdx.x; j < k; j += blockDim.x) lam[j] = 1.f;
}

// the metric into the handle's low-rank block, in k_low_rank_prepare's layout
__global__ void k_lrd_install(int D, int k, const float* __restrict__ sigma, const float* __restrict__ U,
                              const float* __restrict__ lam, float* __restrict__ blk) {
  float* sg = blk + (size_t)D * k;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < D * k; i += gridDim.x * blockDim.x) blk[i] = U[i];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < D) {
    sg[i] = sigma[i];
    sg[D + i] = 1.0f / sigma[i];
  }
  if (i < k) {
    sg[2 * D + i] = lam[i] - 1.0f;
    sg[2 * D + k + i] = 1.0f / sqrtf(lam[i]) - 1.0f;
  }
}

// damping input (:599-634, _low_rank_precondition_pos :215-239): P = (x + ((x U)(lam^-1/2 - 1)) U^T) / sigma with x the
// chain's position minus its fold's mean (the transform is linear, so this is the fold-centred transformed position).
// One warp per chain, the row in registers.
__global__ void k_lrd_transform(int C, int n, int D, int k, const float* __restrict__ q, const float* __restrict__ mu,
                                const float* __restrict__ sigma, const float* __restrict__ U, const float* __restrict__ lam,
                                float* __restrict__ P) {
  const int chain = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (chain >= C) return;
  constexpr int NS = kLrdMaxDim / 32;
  const float* m = mu + (size_t)(chain / n) * D;
  float x[NS], y[NS];
#pragma unroll
  for (int s = 0; s < NS; ++s) {
    const int d = s * 32 + lane;
    x[s] = d < D ? q[(size_t)chain * D + d] - m[d] : 0.f;
    y[s] = x[s];
  }
  for (int j = 0; j < k; ++j) {
    float t = 0.f;
#pragma unroll
    for (int s = 0; s < NS; ++s) {
      const int d = s * 32 + lane;
      if (d < D) t = fmaf(x[s], U[(size_t)d * k + j], t);
    }
    t = warp_sum(t) * (1.0f / sqrtf(lam[j]) - 1.0f);
#pragma unroll
    for (int s = 0; s < NS; ++s) {
      const int d = s * 32 + lane;
      if (d < D) y[s] = fmaf(U[(size_t)d * k + j], t, y[s]);
    }
  }
#pragma unroll
  for (int s = 0; s < NS; ++s) {
    const int d = s * 32 + lane;
    if (d < D) P[(size_t)chain * D + d] = y[s] / sigma[d];
  }
}

static long long next_pow2(long long n) {
  long long p = 1;
  while (p < n) p <<= 1;
  return p;
}

}  // namespace bjx

using namespace bjx;

extern "C" size_t bjx_meads_state_floats(int32_t num_folds, int32_t dim) {
  return (size_t)3 * num_folds + (size_t)3 * num_folds * dim;
}
extern "C" size_t bjx_meads_scratch_floats(int32_t n_chains, int32_t dim, int32_t num_folds) {
  return (size_t)3 * num_folds * dim + (size_t)2 * n_chains + (size_t)2 * num_folds * meads_pairs(dim);
}

extern "C" int bjx_meads_update(bjx_handle_t h, const float* q, const float* grad, int32_t num_folds, int32_t t,
                                float step_size_multiplier, float damping_slowdown, float* state, float* scratch) {
  if (!h || !q || !grad || !state || !scratch) return bjx_fail(h, BJX_E_INVALID, "null argument");
  const int C = h->cfg.n_chains, D = h->cfg.dim, K = num_folds;
  if (K < 1 || K > 64) return bjx_fail(h, BJX_E_INVALID, "num_folds must be in [1, 64]");
  if (C % K != 0) return bjx_fail(h, BJX_E_INVALID, "num_chains must be divisible by num_folds");  // meads_adaptation.py:470-473
  const int n = C / K;
  if (n < 2) return bjx_fail(h, BJX_E_INVALID, "MEADS needs at least 2 chains per fold");
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  float* mu = scratch;
  float* sd = mu + (size_t)K * D;
  float* mus = sd + (size_t)K * D;
  float* rg = mus + (size_t)K * D;
  float* rq = rg + C;
  float* tiles = rq + C;
  const int T = (D + 31) / 32, pairs = meads_pairs(D);
  k_meads_moments<<<dim3(T, K), dim3(32, 8), 0, h->stream>>>(n, D, q, mu, sd, mus);
  k_meads_rows<<<(C + 3) / 4, 128, 0, h->stream>>>(C, n, D, q, grad, sd, mus, rg, rq);
  k_meads_gram<<<dim3(pairs, 2, K), dim3(32, 32), 0, h->stream>>>(n, D, T, q, grad, sd, mus, tiles);
  k_meads_finish<<<1, 256, 0, h->stream>>>(n, D, K, pairs, t, step_size_multiplier, damping_slowdown, sd, rg, rq, tiles, state);
  BJX_CUDA(cudaGetLastError());
  return 0;
}

extern "C" size_t bjx_maximum_eigenvalue_scratch_floats(int64_t n, int32_t d) {
  return (size_t)2 * d + (size_t)2 * n + (size_t)meads_pairs(d);
}

// maximum_eigenvalue (meads_adaptation.py:787-817) of a float32 [n, d] device matrix; out: one device float
extern "C" int bjx_maximum_eigenvalue(bjx_handle_t h, const float* x, int64_t n, int32_t d, float* out, float* scratch) {
  if (!h || !x || !out || !scratch || n < 2 || d < 1 || n > (1ll << 30)) return bjx_fail(h, BJX_E_INVALID, "bad argument");
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  float* ones = scratch;
  float* zeros = ones + d;
  float* rg = zeros + d;
  float* rq = rg + n;
  float* tiles = rq + n;
  const int T = (d + 31) / 32, pairs = meads_pairs(d);
  k_fill2<<<(d + 255) / 256, 256, 0, h->stream>>>(ones, d, 1.0f, zeros, 0.0f);
  k_meads_rows<<<(unsigned)((n + 3) / 4), 128, 0, h->stream>>>((int)n, (int)n, d, x, x, ones, zeros, rg, rq);
  k_meads_gram<<<dim3(pairs, 1, 1), dim3(32, 32), 0, h->stream>>>((int)n, d, T, x, x, ones, zeros, tiles);
  k_maxeig_finish<<<1, 256, 0, h->stream>>>((int)n, pairs, rg, tiles, out);
  BJX_CUDA(cudaGetLastError());
  return 0;
}

extern "C" size_t bjx_permutation_scratch_bytes(int64_t n) { return (size_t)next_pow2(n) * 8 + (size_t)n * 4; }

extern "C" int bjx_permutation(bjx_handle_t h, const uint32_t* key, int64_t fold_index, int64_t n, int32_t* perm_out,
                               void* scratch) {
  if (!h || !key || !perm_out || !scratch || n < 1 || n > (1ll << 30)) return bjx_fail(h, BJX_E_INVALID, "bad argument");
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  const long long np2 = next_pow2(n);
  unsigned long long* comp = (unsigned long long*)scratch;
  int* tmp = (int*)(comp + np2);
  const int rounds = (int)std::ceil(3.0 * std::log((double)std::max<long long>(1, n)) / std::log(4294967295.0));
  // ping-pong so that the last round lands in perm_out
  int* bufs[2] = {perm_out, tmp};
  int cur = (rounds % 2 == 1) ? 0 : 1;
  const int* prev = nullptr;
  const unsigned blocks = (unsigned)((np2 + 255) / 256);
  for (int r = 0; r < rounds; ++r) {
    k_perm_keys<<<blocks, 256, 0, h->stream>>>(key, fold_index, r, (int)n, np2, comp);
    for (long long k = 2; k <= np2; k <<= 1)
      for (long long j = k >> 1; j > 0; j >>= 1) k_bitonic_step<<<blocks, 256, 0, h->stream>>>(comp, np2, j, k);
    k_perm_apply<<<(unsigned)((n + 255) / 256), 256, 0, h->stream>>>(comp, prev, bufs[cur], (int)n);
    prev = bufs[cur];
    cur ^= 1;
  }
  if (n == 1) BJX_CUDA(cudaMemsetAsync(perm_out, 0, 4, h->stream));
  BJX_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int bjx_gather_rows(bjx_handle_t h, const int32_t* perm, const float* src, float* dst, int64_t rows, int32_t width) {
  if (!h || !perm || !src || !dst || rows < 0 || width < 1 || src == dst) return bjx_fail(h, BJX_E_INVALID, "bad argument");
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  if (rows == 0) return 0;
  k_gather_rows<<<(unsigned)((rows + 3) / 4), 128, 0, h->stream>>>(perm, src, dst, (int)rows, width);
  BJX_CUDA(cudaGetLastError());
  return 0;
}

// ---- MEADS-LRD entry points -----------------------------------------------------------------------------------------
extern "C" size_t bjx_meads_lrd_state_floats(int32_t n_chains, int32_t dim, int32_t rank) {
  if (n_chains < 1 || dim < 1 || dim > kLrdMaxDim || rank < 1 || rank > kLrdMaxRank || rank > dim) return 0;
  return lrd_layout(n_chains, dim, rank).total;
}
extern "C" size_t bjx_meads_lrd_scratch_floats(int32_t n_chains, int32_t dim, int32_t num_folds) {
  return bjx_meads_scratch_floats(n_chains, dim, num_folds) + (size_t)2 * num_folds * dim + (size_t)n_chains +
         (size_t)n_chains * dim;
}

// the handle's rank-k low-rank metric (installed once by the caller; the warm-up rewrites it in place)
static int lrd_check(bjx_handle_t h, int& k) {
  const int D = h->cfg.dim;
  if (h->metric_kind != BJX_METRIC_LOW_RANK || !h->lr_block || h->lr_k < 1)
    return bjx_fail(h, BJX_E_UNSUPPORTED, "MEADS-LRD needs a low-rank metric on the handle (bjx_set_metric_low_rank)");
  k = h->lr_k;
  if (D > kLrdMaxDim || k > kLrdMaxRank || k > D)
    return bjx_fail(h, BJX_E_UNSUPPORTED, "MEADS-LRD is built for dim <= 512 and 1 <= rank <= min(16, dim)");
  return 0;
}

static int lrd_eigensolve(bjx_handle_t h, int k, int gate, const LrdLayout& L, float* ls) {
  const int D = h->cfg.dim;
  int rc = eig_smem_opt_in<false>(h);
  if (rc) return rc;
  k_lrd_eig<false><<<kEigCtas, kEigThreads, eig_smem_bytes(D), h->stream>>>(
      D, k, lrd_basis_cols(D, k), gate, ls + L.cm, ls + L.W, ls, ls + L.sigma, ls + L.U, ls + L.lam, ls + L.basis);
  BJX_CHECK_LAUNCH("k_lrd_eig");
  return 0;
}

// the launcher shared with the low-rank window adaptation (bjx_internal.h)
void launch_lrd_install(int D, int k, const float* sigma, const float* U, const float* lam, float* blk, cudaStream_t s) {
  k_lrd_install<<<(D + 255) / 256, 256, 0, s>>>(D, k, sigma, U, lam, blk);
}

extern "C" int bjx_meads_lrd_update(bjx_handle_t h, const float* q, const float* grad, int32_t num_folds, int32_t t,
                                    int32_t in_window, float step_size_multiplier, float damping_slowdown, float* state,
                                    float* lrd_state, float* scratch) {
  if (!h || !q || !grad || !state || !lrd_state || !scratch) return bjx_fail(h, BJX_E_INVALID, "null argument");
  const int C = h->cfg.n_chains, D = h->cfg.dim, K = num_folds;
  if (K < 1 || K > 64) return bjx_fail(h, BJX_E_INVALID, "num_folds must be in [1, 64]");
  if (C % K != 0) return bjx_fail(h, BJX_E_INVALID, "num_chains must be divisible by num_folds");
  const int n = C / K;
  if (n < 2) return bjx_fail(h, BJX_E_INVALID, "MEADS needs at least 2 chains per fold");
  int k = 0;
  int rc = lrd_check(h, k);
  if (rc) return rc;
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  const LrdLayout L = lrd_layout(C, D, k);
  float* ls = lrd_state;
  float* mu = scratch;
  float* sd = mu + (size_t)K * D;
  float* mus = sd + (size_t)K * D;
  float* rg = mus + (size_t)K * D;
  float* rq = rg + C;
  float* tiles = rq + C;
  const int T = (D + 31) / 32, pairs = meads_pairs(D);
  float* ones = tiles + (size_t)2 * K * pairs;
  float* zeros = ones + (size_t)K * D;
  float* rdummy = zeros + (size_t)K * D;
  float* P = rdummy + C;
  cudaStream_t s = h->stream;
  // the fold statistics of bjx_meads_update: the step sizes come from these unchanged.  Only the gradient half of the
  // Gram tiles (grid y = 1) is formed here; the position half comes from the transformed positions below.
  k_meads_moments<<<dim3(T, K), dim3(32, 8), 0, s>>>(n, D, q, mu, sd, mus);
  k_meads_rows<<<(C + 3) / 4, 128, 0, s>>>(C, n, D, q, grad, sd, mus, rg, rq);
  k_meads_gram<<<dim3(pairs, 1, K), dim3(32, 32), 0, s>>>(n, D, T, q, grad, sd, mus, tiles);
  BJX_CHECK_LAUNCH("k_meads_gram");
  // this step's metric (:549-568)
  if (in_window) {
    // k_block_stats also sums an acceptance array over each block; q stands in for it (that sum is not read here)
    launch_block_stats(C, D, q, q, ls + L.stats, s);
    launch_cov_fold(C, D, q, ls + L.stats, ls + L.cov, s);
    launch_cov_merge(cov_stat_blocks(C), D, ls + L.cov, nullptr, ls + L.W, ls + L.cm, s);
    BJX_CHECK_LAUNCH("launch_cov_merge");
  }
  k_lrd_fallback<<<1, 512, 0, s>>>(D, k, K, n, mu, sd, in_window ? 1 : 0, ls + L.cm, ls, ls + L.sigma, ls + L.U, ls + L.lam);
  BJX_CHECK_LAUNCH("k_lrd_fallback");
  if (in_window) {
    rc = lrd_eigensolve(h, k, 1, L, ls);
    if (rc) return rc;
  }
  k_lrd_install<<<(D + 255) / 256, 256, 0, s>>>(D, k, ls + L.sigma, ls + L.U, ls + L.lam, h->lr_block);
  // damping from the fold-centred, low-rank-preconditioned positions (:599-634): their statistics replace the position
  // half of the fold statistics (rows of X X^T, and the tiles at offset `pairs`) with unit scales and zero means
  k_lrd_transform<<<(C + 7) / 8, 256, 0, s>>>(C, n, D, k, q, mu, ls + L.sigma, ls + L.U, ls + L.lam, P);
  k_fill2<<<(K * D + 255) / 256, 256, 0, s>>>(ones, K * D, 1.0f, zeros, 0.0f);
  k_meads_rows<<<(C + 3) / 4, 128, 0, s>>>(C, n, D, P, P, ones, zeros, rdummy, rq);
  k_meads_gram<<<dim3(pairs, 1, K), dim3(32, 32), 0, s>>>(n, D, T, P, P, ones, zeros, tiles + pairs);
  k_meads_finish<<<1, 256, 0, s>>>(n, D, K, pairs, t, step_size_multiplier, damping_slowdown, sd, rg, rq, tiles, state);
  BJX_CHECK_LAUNCH("k_meads_finish");
  return 0;
}

extern "C" int bjx_meads_lrd_metric(bjx_handle_t h, float* lrd_state, const float* final_q, float* sigma_out, float* U_out,
                                    float* lam_out) {
  if (!h || !lrd_state || !final_q || !sigma_out || !U_out || !lam_out) return bjx_fail(h, BJX_E_INVALID, "null argument");
  int k = 0;
  int rc = lrd_check(h, k);
  if (rc) return rc;
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  const int C = h->cfg.n_chains, D = h->cfg.dim;
  if (C < 2) return bjx_fail(h, BJX_E_INVALID, "MEADS-LRD needs at least 2 chains");
  const LrdLayout L = lrd_layout(C, D, k);
  float* ls = lrd_state;
  float* fin = ls + L.fin;
  cudaStream_t s = h->stream;
  // the last accumulator if it holds 2 D samples, else the fallback on the final positions (:746-771)
  k_meads_moments<<<dim3((D + 31) / 32, 1), dim3(32, 8), 0, s>>>(C, D, final_q, fin, fin + D, fin + 2 * D);
  launch_cov_merge(cov_stat_blocks(C), D, ls + L.cov, nullptr, ls + L.W, ls + L.cm, s);
  k_lrd_fallback<<<1, 512, 0, s>>>(D, k, 1, C, fin, fin + D, 1, ls + L.cm, ls, ls + L.sigma, ls + L.U, ls + L.lam);
  BJX_CHECK_LAUNCH("k_lrd_fallback");
  rc = lrd_eigensolve(h, k, 1, L, ls);
  if (rc) return rc;
  BJX_CUDA(cudaMemcpyAsync(sigma_out, ls + L.sigma, (size_t)D * sizeof(float), cudaMemcpyDeviceToDevice, s));
  BJX_CUDA(cudaMemcpyAsync(U_out, ls + L.U, (size_t)D * k * sizeof(float), cudaMemcpyDeviceToDevice, s));
  BJX_CUDA(cudaMemcpyAsync(lam_out, ls + L.lam, (size_t)k * sizeof(float), cudaMemcpyDeviceToDevice, s));
  return 0;
}
