// Low-rank window adaptation (window_adaptation_low_rank, blackjax/adaptation/low_rank_adaptation.py:458-652 with
// buffer_policy="reset"), pooled over chains: ONE step size and ONE low-rank metric M^-1 = D_s (I + U (Lam - I) U^T) D_s
// for all chains of one GPU.
//
// Per warm-up step (schedule byte = stage | window_end << 1 | retained << 2):
//  - dual averaging on the mean acceptance rate of all chains (pooled_step_size_update, bjx_pooled_step.cuh), fed by the
//    k_block_stats records of the positions;
//  - on a retained slow step the positions and the gradients of all chains are folded into two windowed covariance
//    accumulators (k_cov_syrk / cgl_update_batch, per statistic block).  The reference keeps a circular buffer of the last
//    B draws of the window (metric_recipes.py:601-700); the host knows the schedule, so it marks as retained exactly the
//    steps that buffer still holds at the window end.  Every slow step counts towards n = C x steps of the window, which
//    the estimator divides by whether or not the step is retained (metric_estimators.py:709-721).
//  - at a window end, the estimator (_compute_low_rank_metric, metric_estimators.py:618-808) from the accumulators,
//    with no host round trip:
//      k_lw_merge    Chan merge of the block accumulators in global block order: count c, mean, M2 [D, D] of x and g;
//      k_lw_sigma    x_bar = (c / n) mean, the scatter correction M2 + c d d^T with d = mean - x_bar, population
//                    variances, sigma = clip((var_x / max(var_g, 1e-10))^(1/4), 1e-20, 1e20), mu* = x_bar + sigma^2 g_bar;
//      k_lw_scatter  S_x = D_s^-1 (.) D_s^-1 and S_a = D_s (.) D_s in float32 for the eigensolver (D > 2k only);
//      k_lrd_eig<true> (bjx_meads.cu) twice: the top k eigenvectors of S_x and S_a (the right singular vectors of the
//                    reference's thin SVD), each warm-started from the previous window's Ritz basis;
//      k_lw_final    one CTA, float64: Q = orth([U_x, U_a]) by twice-repeated modified Gram-Schmidt (Q = I when
//                    D <= 2k: the result does not depend on the basis of the span), C_x = Q^T S_x Q / gamma + I and
//                    C_a likewise with S_x, S_a re-formed in float64 from the float32 M2, Sigma = spd_mean(C_x, C_a^-1)
//                    with both spectra floored at eps max|lam| (metric_estimators.py:77-142), eigh(Sigma) floored, the
//                    top min(k, q) pairs by |lam - 1|, lam = 1 inside [1/cutoff, cutoff], zero / one padding;
//      k_lrd_install (bjx_meads.cu) rewrites the handle's low-rank block in place; the accumulators are reset and dual
//                    averaging restarts at exp(log_step_avg) (staged_adaptation.py:233-249).
// Every reduction runs in a fixed order: two runs are bit-identical.
#include <cmath>

#include "bjx_handle.h"
#include "bjx_internal.h"
#include "bjx_lrd_eig.cuh"
#include "bjx_pooled_step.cuh"

namespace bjx {
namespace {

constexpr int kLwHdr = 64;          // scalar slots | eigensolver header of S_x | eigensolver header of S_a
constexpr int kLwMaxDim = 512, kLwMaxRank = 16, kQ = 2 * kLwMaxRank;
constexpr int kJacobiSweepsD = 40;
// header slots after PS_* (bjx_pooled_step.cuh): slow steps of the open window, windows ended
enum { LW_LEN = 8, LW_WINDOWS };
constexpr int kEhx = 32, kEha = 48;  // LRD_* slots of the two solves (include/bjx.h)

size_t even(size_t n) { return (n + 1) & ~(size_t)1; }

size_t lrd_eig_basis_floats(int D, int k) { return (size_t)D * lrd_basis_cols(D, k); }

struct LwLayout {
  size_t sigma, U, lam, mu, ux, lx, ua, la, bx, ba, stx, stg, covx, covg, m2x, m2g, cmx, cmg, sx, sa, dbl, total;
  size_t Sc;  // floats per block accumulator
  int nb;
};
// state: header | sigma[D] U[D,k] lam[k] mu*[D] (the current metric) | the two solves' U [D,k], lam [k] and Ritz bases |
// k_block_stats records of q and g | block accumulators of q and g | merged M2 of q and g [D,D] | merged (count, mean) |
// S_x, S_a float32 [D,D] (D > 2k) | float64: sigma[D] d_x[D] d_g[D] Q[D,32] T[D,32] scale[D] u[D]
LwLayout lw_layout(int C, int D, int k) {
  LwLayout L{};
  const size_t d = (size_t)D, sc = cov_block_floats(D);
  const bool solve = D > 2 * k;
  L.nb = cov_stat_blocks(C);
  L.Sc = sc;
  size_t o = kLwHdr;
  L.sigma = o; o += d;
  L.U = o; o += d * k;
  L.lam = o; o += k;
  L.mu = o; o += d;
  L.ux = o; o += d * k;
  L.lx = o; o += k;
  L.ua = o; o += d * k;
  L.la = o; o += k;
  L.bx = o; o += solve ? lrd_eig_basis_floats(D, k) : 0;
  L.ba = o; o += solve ? lrd_eig_basis_floats(D, k) : 0;
  L.stx = o; o += (size_t)L.nb * (2 + 2 * d);
  L.stg = o; o += (size_t)L.nb * (2 + 2 * d);
  L.covx = o; o += (size_t)L.nb * sc;
  L.covg = o; o += (size_t)L.nb * sc;
  L.m2x = o; o += d * d;
  L.m2g = o; o += d * d;
  L.cmx = o; o += 1 + d;
  L.cmg = o; o += 1 + d;
  L.sx = o; o += solve ? d * d : 0;
  L.sa = o; o += solve ? d * d : 0;
  L.dbl = even(o); o = L.dbl + 2 * (5 * d + 2 * d * kQ);
  L.total = o;
  return L;
}

__global__ void k_lw_init(int D, int k, float* __restrict__ st, float eps0, const LwLayout L) {
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    st[L.sigma + d] = 1.f;
    st[L.mu + d] = 0.f;
    for (int j = 0; j < k; ++j) st[L.U + (size_t)d * k + j] = 0.f;
  }
  for (int j = threadIdx.x; j < k; j += blockDim.x) st[L.lam + j] = 1.f;
  if (threadIdx.x == 0) {
    da_init(st + PS_DA, eps0);
    st[PS_EPS] = da_step_size(st + PS_DA);
  }
}

// the pooled step-size update and the window's step count
__global__ void k_lw_adapt(int nblk, const float* __restrict__ blocks, size_t S, float* __restrict__ st, int stage,
                           int window_end, float target, float* __restrict__ eps_hist) {
  if (threadIdx.x != 0) return;
  pooled_step_size_update(nblk, blocks, S, st, window_end, target, eps_hist);
  if (stage) st[LW_LEN] += 1.f;
}

// grid (ceil(D / 256), D, 2): the block accumulators of x (z = 0) or g (z = 1) merged in global block order; raw M2, both
// halves, and (count, mean) -- k_cov_merge_whiten's arithmetic without the division
__global__ void k_lw_merge(int D, int nblk, const float* __restrict__ covx, const float* __restrict__ covg, size_t cstride,
                           float* __restrict__ m2x, float* __restrict__ m2g, float* __restrict__ cmx, float* __restrict__ cmg) {
  const int i = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j > i) return;
  const float* cov = blockIdx.z ? covg : covx;
  float* out = blockIdx.z ? m2g : m2x;
  float* cm = blockIdx.z ? cmg : cmx;
  float n = 0.f, mi = 0.f, mj = 0.f, m2 = 0.f;
  for (int b = 0; b < nblk; ++b) {
    const float* blk = cov + (size_t)b * cstride;
    if (blk[0] == 0.f) continue;
    float fm, fc, nab;
    cgl_factors(n, blk[0], fm, fc, nab);
    const float di = blk[2 + i] - mi, dj = blk[2 + j] - mj;
    m2 = m2 + blk[2 + D + (size_t)i * D + j] + di * dj * fc;
    mi = mi + di * fm;
    mj = mj + dj * fm;
    n = nab;
  }
  if (j == 0) { cm[0] = n; cm[1 + i] = mi; }
  out[(size_t)i * D + j] = m2;
  out[(size_t)j * D + i] = m2;
}

// sigma, mu*, the scatter corrections (metric_estimators.py:709-727): float64 from here on
__global__ void k_lw_sigma(int D, double c_total, const float* __restrict__ st_hdr, const float* __restrict__ m2x,
                           const float* __restrict__ m2g, const float* __restrict__ cmx, const float* __restrict__ cmg,
                           float* __restrict__ sigma, float* __restrict__ mu_star, double* __restrict__ sig_d,
                           double* __restrict__ dx, double* __restrict__ dg) {
  const double n = c_total * (double)st_hdr[LW_LEN];
  const double n_safe = fmax(n, 2.0), c = (double)cmx[0];
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    const double mx = cmx[1 + d], mg = cmg[1 + d];
    const double xbar = c * mx / n_safe, gbar = c * mg / n_safe;
    const double ex = mx - xbar, eg = mg - gbar;
    const double vx = ((double)m2x[(size_t)d * D + d] + c * ex * ex) / n_safe;
    const double vg = ((double)m2g[(size_t)d * D + d] + c * eg * eg) / n_safe;
    double s = pow(fmax(vx / fmax(vg, 1e-10), 0.0), 0.25);
    s = fmin(fmax(s, 1e-20), 1e20);
    sig_d[d] = s;
    dx[d] = ex;
    dg[d] = eg;
    sigma[d] = (float)s;
    mu_star[d] = (float)(xbar + s * s * gbar);
  }
}

__device__ __forceinline__ double lw_sx(int D, const float* m2x, double c, const double* sig, const double* dx, int r, int q) {
  return ((double)m2x[(size_t)r * D + q] + c * dx[r] * dx[q]) / (sig[r] * sig[q]);
}
__device__ __forceinline__ double lw_sa(int D, const float* m2g, double c, const double* sig, const double* dg, int r, int q) {
  return ((double)m2g[(size_t)r * D + q] + c * dg[r] * dg[q]) * (sig[r] * sig[q]);
}

// grid (ceil(D / 256), D): S_x and S_a in float32 for the eigensolver
__global__ void k_lw_scatter(int D, const float* __restrict__ m2x, const float* __restrict__ m2g, const float* __restrict__ cmx,
                             const double* __restrict__ sig, const double* __restrict__ dx, const double* __restrict__ dg,
                             float* __restrict__ sx, float* __restrict__ sa) {
  const int i = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= D) return;
  const double c = (double)cmx[0];
  sx[(size_t)i * D + j] = (float)lw_sx(D, m2x, c, sig, dx, i, j);
  sa[(size_t)i * D + j] = (float)lw_sa(D, m2g, c, sig, dg, i, j);
}

constexpr int kFinThreads = 1024;

// block-wide float64 sum in a fixed order (32 warps, then one)
__device__ double lw_block_sum(double v, double* red) {
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  double s = 0.0;
  for (int i = 0; i < kFinThreads / 32; ++i) s += red[i];
  return s;
}

// cyclic Jacobi eigh of the symmetric n x n matrix M (stride kQ, n <= kQ; destroyed) -> eigenvalues w[n] (unordered),
// eigenvectors in the columns of V.  Round-robin ordering, n2 / 2 disjoint rotations per round; a pair is rotated while
// |m_pq| > 1e-17 sqrt|m_pp m_qq| and the sweeps stop once none is -- the relative criterion, so that the small
// eigenvalues of a matrix spanning many orders of magnitude keep their accuracy.
__device__ void lw_jacobi(double* M, double* V, double* w, int n, double* cs, int* flag) {
  const int tid = threadIdx.x;
  const int n2 = n + (n & 1), half = n2 / 2;
  for (int e = tid; e < kQ * kQ; e += blockDim.x) {
    const int i = e / kQ, j = e - i * kQ;
    V[e] = i == j ? 1.0 : 0.0;
    if (i >= n || j >= n) M[e] = 0.0;
  }
  __syncthreads();
  auto pair_of = [&](int m, int rd, int& p, int& q) {
    if (m == 0) { p = rd % (n2 - 1); q = n2 - 1; }
    else { p = (rd + m) % (n2 - 1); q = (rd - m + n2 - 1) % (n2 - 1); }
  };
  if (n2 < 2) return;
  for (int sweep = 0; sweep < kJacobiSweepsD; ++sweep) {
    if (tid == 0) flag[0] = 1;
    __syncthreads();
    for (int rd = 0; rd < n2 - 1; ++rd) {
      if (tid < half) {
        int p, q;
        pair_of(tid, rd, p, q);
        const double app = M[p * kQ + p], aqq = M[q * kQ + q], apq = M[p * kQ + q];
        double c = 1.0, s = 0.0;
        if (fabs(apq) > 1e-17 * sqrt(fabs(app * aqq)) && apq != 0.0) {
          const double tau = (aqq - app) / (2.0 * apq);
          const double t = (tau >= 0.0 ? 1.0 : -1.0) / (fabs(tau) + sqrt(1.0 + tau * tau));
          c = 1.0 / sqrt(1.0 + t * t);
          s = t * c;
          flag[0] = 0;
        }
        cs[tid] = c;
        cs[kQ + tid] = s;
      }
      __syncthreads();
      for (int e = tid; e < half * n2; e += blockDim.x) {  // rows p, q
        const int m = e / n2, col = e - m * n2;
        int p, q;
        pair_of(m, rd, p, q);
        const double c = cs[m], s = cs[kQ + m], x = M[p * kQ + col], y = M[q * kQ + col];
        M[p * kQ + col] = c * x - s * y;
        M[q * kQ + col] = s * x + c * y;
      }
      __syncthreads();
      for (int e = tid; e < half * n2; e += blockDim.x) {  // columns p, q, and the eigenvectors
        const int m = e / n2, row = e - m * n2;
        int p, q;
        pair_of(m, rd, p, q);
        const double c = cs[m], s = cs[kQ + m];
        double x = M[row * kQ + p], y = M[row * kQ + q];
        M[row * kQ + p] = c * x - s * y;
        M[row * kQ + q] = s * x + c * y;
        x = V[row * kQ + p]; y = V[row * kQ + q];
        V[row * kQ + p] = c * x - s * y;
        V[row * kQ + q] = s * x + c * y;
      }
      __syncthreads();
    }
    const bool done = flag[0] != 0;
    __syncthreads();
    if (done) break;
  }
  for (int j = tid; j < n; j += blockDim.x) w[j] = M[j * kQ + j];
  __syncthreads();
}

// max(v, eps max|v|) over v[n] (_relative_pd_floor, float64)
__device__ void lw_floor(double* v, int n) {
  __syncthreads();
  double mx = 0.0;
  for (int j = 0; j < n; ++j) mx = fmax(mx, fabs(v[j]));
  const double fl = 2.220446049250313e-16 * fmax(mx, 2.2250738585072014e-308);
  __syncthreads();
  for (int j = threadIdx.x; j < n; j += blockDim.x) v[j] = fmax(v[j], fl);
  __syncthreads();
}

// one CTA: Q, the projections, the SPD mean, eigh, selection and masking (see the top of the file)
__global__ void __launch_bounds__(kFinThreads) k_lw_final(int D, int k, float gamma, float cutoff, const float* __restrict__ m2x,
                                                           const float* __restrict__ m2g, const float* __restrict__ cmx,
                                                           const float* __restrict__ ux, const float* __restrict__ ua,
                                                           const double* __restrict__ sig, const double* __restrict__ dx,
                                                           const double* __restrict__ dg, double* __restrict__ Qg,
                                                           double* __restrict__ Tg, double* __restrict__ scl,
                                                           double* __restrict__ us, float* __restrict__ U_out,
                                                           float* __restrict__ lam_out, float* __restrict__ hdr) {
  __shared__ double A0[kQ * kQ], A1[kQ * kQ], A2[kQ * kQ], A3[kQ * kQ], A4[kQ * kQ];
  __shared__ double wa[kQ], wb[kQ], wc[kQ], cs[2 * kQ], red[32];
  __shared__ int order[kQ], flag[2];
  const int tid = threadIdx.x, NT = blockDim.x;
  const bool solve = D > 2 * k;
  const int q = solve ? 2 * k : D;
  const double c = (double)cmx[0];

  // ---- Q [D, q] (row-major, stride kQ) ----
  if (!solve) {
    for (int e = tid; e < D * kQ; e += NT) Qg[e] = (e / kQ == e % kQ) ? 1.0 : 0.0;
    __syncthreads();
  } else {
    for (int j = 0; j < q; ++j) {
      for (int cand = -1; cand < D; ++cand) {  // the column itself, else e_0, e_1, ... until one is independent
        for (int r = tid; r < D; r += NT)
          Qg[(size_t)r * kQ + j] = cand < 0 ? (double)(j < k ? ux[(size_t)r * k + j] : ua[(size_t)r * k + j - k])
                                            : (r == cand ? 1.0 : 0.0);
        __syncthreads();
        double nrm0 = 0.0;
        {
          double a = 0.0;
          for (int r = tid; r < D; r += NT) a += Qg[(size_t)r * kQ + j] * Qg[(size_t)r * kQ + j];
          nrm0 = sqrt(lw_block_sum(a, red));
        }
        for (int pass = 0; pass < 2; ++pass)  // modified Gram-Schmidt, twice
          for (int i = 0; i < j; ++i) {
            double a = 0.0;
            for (int r = tid; r < D; r += NT) a += Qg[(size_t)r * kQ + i] * Qg[(size_t)r * kQ + j];
            const double h = lw_block_sum(a, red);
            __syncthreads();
            for (int r = tid; r < D; r += NT) Qg[(size_t)r * kQ + j] -= h * Qg[(size_t)r * kQ + i];
            __syncthreads();
          }
        double a = 0.0;
        for (int r = tid; r < D; r += NT) a += Qg[(size_t)r * kQ + j] * Qg[(size_t)r * kQ + j];
        const double nrm = sqrt(lw_block_sum(a, red));
        if (nrm > 1e-6 * nrm0 && nrm > 0.0) {
          __syncthreads();
          for (int r = tid; r < D; r += NT) Qg[(size_t)r * kQ + j] /= nrm;
          __syncthreads();
          break;
        }
        __syncthreads();
      }
    }
  }

  // ---- C = Q^T S Q / gamma + I for S_x (A0) and S_a (A1); T = S Q in global memory, with
  // S = D (M2 + c d d^T) D = M2 * scale scale^T + c u u^T, D = diag(scale), u = D d ----
  for (int which = 0; which < 2; ++which) {
    double* Cm = which ? A1 : A0;
    const float* m2 = which ? m2g : m2x;
    for (int r = tid; r < D; r += NT) {
      const double f = which ? sig[r] : 1.0 / sig[r];
      scl[r] = f;
      us[r] = (which ? dg[r] : dx[r]) * f;
    }
    __syncthreads();
    for (int e = tid; e < D * q; e += NT) {
      const int r = e / q, j = e - r * q;
      const double fr = scl[r], ur = c * us[r];
      double s = 0.0;
      for (int cc = 0; cc < D; ++cc) {
        const double v = (double)m2[(size_t)r * D + cc] * fr * scl[cc] + ur * us[cc];
        s = fma(v, Qg[(size_t)cc * kQ + j], s);
      }
      Tg[(size_t)r * kQ + j] = s;
    }
    __syncthreads();
    for (int e = tid; e < q * q; e += NT) {
      const int i = e / q, j = e - i * q;
      double s = 0.0;
      for (int r = 0; r < D; ++r) s = fma(Qg[(size_t)r * kQ + i], Tg[(size_t)r * kQ + j], s);
      A2[i * kQ + j] = s;
    }
    __syncthreads();
    for (int e = tid; e < q * q; e += NT) {
      const int i = e / q, j = e - i * q;
      Cm[i * kQ + j] = 0.5 * (A2[i * kQ + j] + A2[j * kQ + i]) / (double)gamma + (i == j ? 1.0 : 0.0);
    }
    __syncthreads();
  }

  // ---- Sigma = spd_mean(C_x, B) with B = C_a^-1: B's eigenpairs are (1 / lam, v) of C_a ----
  lw_jacobi(A1, A2, wa, q, cs, flag);                 // C_a -> vecs_b in A2, 1 / vals_b in wa
  for (int j = tid; j < q; j += NT) wa[j] = 1.0 / wa[j];
  lw_floor(wa, q);                                    // vals_b
  for (int e = tid; e < q * q; e += NT) {             // tmp = vecs_b^T C_x vecs_b -> A3 (via A1 = C_x vecs_b)
    const int i = e / q, j = e - i * q;
    double s = 0.0;
    for (int t = 0; t < q; ++t) s = fma(A0[i * kQ + t], A2[t * kQ + j], s);
    A1[i * kQ + j] = s;
  }
  __syncthreads();
  for (int e = tid; e < q * q; e += NT) {
    const int i = e / q, j = e - i * q;
    double s = 0.0;
    for (int t = 0; t < q; ++t) s = fma(A2[t * kQ + i], A1[t * kQ + j], s);
    A3[i * kQ + j] = s / (sqrt(wa[i]) * sqrt(wa[j]));  // M = inv_sqrt_b tmp inv_sqrt_b
  }
  __syncthreads();
  for (int e = tid; e < q * q; e += NT) {             // symmetrise M
    const int i = e / q, j = e - i * q;
    if (i < j) {
      const double m = 0.5 * (A3[i * kQ + j] + A3[j * kQ + i]);
      A3[i * kQ + j] = m;
      A3[j * kQ + i] = m;
    }
  }
  __syncthreads();
  lw_jacobi(A3, A4, wb, q, cs, flag);                 // vecs_m in A4, vals_m in wb
  lw_floor(wb, q);
  for (int e = tid; e < q * q; e += NT) {             // W = vecs_b diag(sqrt_b) vecs_m -> A0
    const int i = e / q, j = e - i * q;
    double s = 0.0;
    for (int t = 0; t < q; ++t) s = fma(A2[i * kQ + t] * sqrt(wa[t]), A4[t * kQ + j], s);
    A0[i * kQ + j] = s;
  }
  __syncthreads();
  for (int e = tid; e < q * q; e += NT) {             // Sigma = (W sqrt_m) W^T -> A1
    const int i = e / q, j = e - i * q;
    double s = 0.0;
    for (int t = 0; t < q; ++t) s = fma(A0[i * kQ + t] * sqrt(wb[t]), A0[j * kQ + t], s);
    A1[i * kQ + j] = s;
  }
  __syncthreads();
  for (int e = tid; e < q * q; e += NT) {
    const int i = e / q, j = e - i * q;
    if (i < j) {
      const double m = 0.5 * (A1[i * kQ + j] + A1[j * kQ + i]);
      A1[i * kQ + j] = m;
      A1[j * kQ + i] = m;
    }
  }
  __syncthreads();
  lw_jacobi(A1, A3, wc, q, cs, flag);                 // eigh(Sigma): vecs in A3, vals in wc
  lw_floor(wc, q);

  // ---- selection: eigh's ascending order, then a stable argsort of -|lam - 1| ----
  const int r_act = k < q ? k : q;
  if (tid == 0) {
    for (int j = 0; j < q; ++j) order[j] = j;
    for (int m = 1; m < q; ++m)  // insertion sort, ascending eigenvalue (stable)
      for (int j = m; j > 0 && wc[order[j]] < wc[order[j - 1]]; --j) { const int t = order[j]; order[j] = order[j - 1]; order[j - 1] = t; }
    for (int m = 1; m < q; ++m)  // insertion sort, descending |lam - 1| (stable)
      for (int j = m; j > 0 && fabs(wc[order[j]] - 1.0) > fabs(wc[order[j - 1]] - 1.0); --j) {
        const int t = order[j]; order[j] = order[j - 1]; order[j - 1] = t;
      }
  }
  __syncthreads();
  for (int e = tid; e < D * k; e += NT) {
    const int r = e / k, m = e - r * k;
    double s = 0.0;
    if (m < r_act)
      for (int t = 0; t < q; ++t) s = fma(Qg[(size_t)r * kQ + t], A3[t * kQ + order[m]], s);
    U_out[e] = (float)s;
  }
  for (int m = tid; m < k; m += NT) {
    double l = 1.0;
    if (m < r_act) {
      const double v = wc[order[m]];
      l = (v < 1.0 / (double)cutoff || v > (double)cutoff) ? v : 1.0;
    }
    lam_out[m] = (float)l;
  }
  if (tid == 0) {
    hdr[LW_LEN] = 0.f;
    hdr[LW_WINDOWS] += 1.f;
  }
}

// k_lrd_eig in its scatter mode on the symmetric W [D, D]: the top k eigenpairs by the largest eigenvalue into U [D, k]
// (columns descending) and lam [k], warm-started from basis once hdr[LRD_WARM] is set
int launch_lrd_eig_scatter(bjx_handle_t h, int D, int k, const float* W, float* hdr, float* U, float* lam, float* basis) {
  int rc = eig_smem_opt_in<true>(h);
  if (rc) return rc;
  k_lrd_eig<true><<<kEigCtas, kEigThreads, eig_smem_bytes(D), h->stream>>>(D, k, lrd_basis_cols(D, k), 1, nullptr, W, hdr,
                                                                           nullptr, U, lam, basis);
  BJX_CHECK_LAUNCH("k_lrd_eig");
  return 0;
}

int lw_check(bjx_handle_t h, int& k) {
  if (h->metric_kind != BJX_METRIC_LOW_RANK || !h->lr_block || h->lr_k < 1)
    return bjx_fail(h, BJX_E_UNSUPPORTED,
                    "the low-rank window adaptation needs a low-rank metric on the handle (bjx_set_metric_low_rank)");
  k = h->lr_k;
  if (h->cfg.dim > kLwMaxDim || k > kLwMaxRank)
    return bjx_fail(h, BJX_E_UNSUPPORTED, "the low-rank window adaptation is built for dim <= 512 and 1 <= rank <= 16");
  return 0;
}

}  // namespace
}  // namespace bjx

using namespace bjx;

extern "C" size_t bjx_lowrank_window_state_floats(int32_t n_chains, int32_t dim, int32_t rank) {
  if (n_chains < 1 || dim < 1 || dim > kLwMaxDim || rank < 1 || rank > kLwMaxRank) return 0;
  return lw_layout(n_chains, dim, rank).total;
}

extern "C" int bjx_lowrank_window_init(bjx_handle_t h, float* state, float initial_step_size, float* step_size_chain_out) {
  if (!h || !state || !step_size_chain_out) return bjx_fail(h, BJX_E_INVALID, "null argument");
  if (!(initial_step_size > 0.f)) return bjx_fail(h, BJX_E_INVALID, "initial_step_size must be positive");
  int k = 0;
  int rc = lw_check(h, k);
  if (rc) return rc;
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  const int C = h->cfg.n_chains, D = h->cfg.dim;
  const LwLayout L = lw_layout(C, D, k);
  BJX_CUDA(cudaMemsetAsync(state, 0, L.total * sizeof(float), h->stream));
  k_lw_init<<<1, 256, 0, h->stream>>>(D, k, state, initial_step_size, L);
  launch_fill_from(C, state + PS_EPS, step_size_chain_out, h->stream);
  BJX_CHECK_LAUNCH("k_lw_init");
  launch_lrd_install(D, k, state + L.sigma, state + L.U, state + L.lam, h->lr_block, h->stream);
  BJX_CHECK_LAUNCH("k_lrd_install");
  return 0;
}

extern "C" int bjx_lowrank_window_update(bjx_handle_t h, float* state, const float* q, const float* grad,
                                         const float* acceptance_rate, int32_t schedule, float target_acceptance, float gamma,
                                         float cutoff, float* step_size_chain, float* eps_history) {
  if (!h || !state || !q || !grad || !acceptance_rate || !step_size_chain) return bjx_fail(h, BJX_E_INVALID, "null argument");
  const int stage = schedule & 1, window_end = (schedule >> 1) & 1, retained = (schedule >> 2) & 1;
  if ((window_end || retained) && !stage) return bjx_fail(h, BJX_E_INVALID, "window ends and retained steps are slow-stage steps");
  if (window_end && !retained) return bjx_fail(h, BJX_E_INVALID, "a window's last step is always retained");
  if (!(gamma > 0.f) || !(cutoff > 0.f)) return bjx_fail(h, BJX_E_INVALID, "gamma and cutoff must be positive");
  int k = 0;
  int rc = lw_check(h, k);
  if (rc) return rc;
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  const int C = h->cfg.n_chains, D = h->cfg.dim;
  const LwLayout L = lw_layout(C, D, k);
  cudaStream_t s = h->stream;
  float* st = state;
  launch_block_stats(C, D, q, acceptance_rate, st + L.stx, s);
  BJX_CHECK_LAUNCH("k_block_stats");
  if (retained) {
    // k_block_stats also sums an acceptance array over each block; grad stands in for it (that sum is not read here)
    launch_block_stats(C, D, grad, grad, st + L.stg, s);
    launch_cov_fold(C, D, q, st + L.stx, st + L.covx, s);
    launch_cov_fold(C, D, grad, st + L.stg, st + L.covg, s);
    BJX_CHECK_LAUNCH("k_cov_syrk");
  }
  k_lw_adapt<<<1, 32, 0, s>>>(L.nb, st + L.stx, 2 + 2 * (size_t)D, st, stage, window_end, target_acceptance, eps_history);
  launch_fill_from(C, st + PS_EPS, step_size_chain, s);
  BJX_CHECK_LAUNCH("k_lw_adapt");
  if (!window_end) return 0;
  double* dbl = reinterpret_cast<double*>(st + L.dbl);
  double* sig = dbl;
  double* dx = sig + D;
  double* dg = dx + D;
  double* Qg = dg + D;
  double* Tg = Qg + (size_t)D * kQ;
  double* scl = Tg + (size_t)D * kQ;
  double* us = scl + D;
  k_lw_merge<<<dim3((D + 255) / 256, D, 2), 256, 0, s>>>(D, L.nb, st + L.covx, st + L.covg, L.Sc, st + L.m2x, st + L.m2g,
                                                          st + L.cmx, st + L.cmg);
  k_lw_sigma<<<1, 512, 0, s>>>(D, (double)C, st, st + L.m2x, st + L.m2g, st + L.cmx, st + L.cmg, st + L.sigma, st + L.mu,
                               sig, dx, dg);
  BJX_CHECK_LAUNCH("k_lw_sigma");
  if (D > 2 * k) {
    k_lw_scatter<<<dim3((D + 255) / 256, D), 256, 0, s>>>(D, st + L.m2x, st + L.m2g, st + L.cmx, sig, dx, dg, st + L.sx, st + L.sa);
    BJX_CHECK_LAUNCH("k_lw_scatter");
    rc = launch_lrd_eig_scatter(h, D, k, st + L.sx, st + kEhx, st + L.ux, st + L.lx, st + L.bx);
    if (rc) return rc;
    rc = launch_lrd_eig_scatter(h, D, k, st + L.sa, st + kEha, st + L.ua, st + L.la, st + L.ba);
    if (rc) return rc;
  }
  k_lw_final<<<1, kFinThreads, 0, s>>>(D, k, gamma, cutoff, st + L.m2x, st + L.m2g, st + L.cmx, st + L.ux, st + L.ua, sig, dx,
                                       dg, Qg, Tg, scl, us, st + L.U, st + L.lam, st);
  BJX_CHECK_LAUNCH("k_lw_final");
  launch_lrd_install(D, k, st + L.sigma, st + L.U, st + L.lam, h->lr_block, s);
  BJX_CHECK_LAUNCH("k_lrd_install");
  // reset: the next window starts with empty accumulators (metric_recipes.py:689-698)
  BJX_CUDA(cudaMemsetAsync(st + L.covx, 0, 2 * (size_t)L.nb * L.Sc * sizeof(float), s));
  return 0;
}

extern "C" int bjx_lowrank_window_final(bjx_handle_t h, const float* state, float* step_size_out, float* mu_star_out,
                                        float* sigma_out, float* U_out, float* lam_out) {
  if (!h || !state || !step_size_out || !mu_star_out || !sigma_out || !U_out || !lam_out)
    return bjx_fail(h, BJX_E_INVALID, "null argument");
  int k = 0;
  int rc = lw_check(h, k);
  if (rc) return rc;
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  const int C = h->cfg.n_chains, D = h->cfg.dim;
  const LwLayout L = lw_layout(C, D, k);
  cudaStream_t s = h->stream;
  launch_da(3, 1, const_cast<float*>(state) + PS_DA, nullptr, 0.f, step_size_out, s);  // exp(log_step_avg)
  BJX_CHECK_LAUNCH("k_da_final");
  BJX_CUDA(cudaMemcpyAsync(mu_star_out, state + L.mu, (size_t)D * sizeof(float), cudaMemcpyDeviceToDevice, s));
  BJX_CUDA(cudaMemcpyAsync(sigma_out, state + L.sigma, (size_t)D * sizeof(float), cudaMemcpyDeviceToDevice, s));
  BJX_CUDA(cudaMemcpyAsync(U_out, state + L.U, (size_t)D * k * sizeof(float), cudaMemcpyDeviceToDevice, s));
  BJX_CUDA(cudaMemcpyAsync(lam_out, state + L.lam, (size_t)k * sizeof(float), cudaMemcpyDeviceToDevice, s));
  return 0;
}
