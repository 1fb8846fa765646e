// The cluster eigensolver of MEADS-LRD (bjx_meads.cu), also run by the low-rank window adaptation
// (bjx_lowrank_window.cu) in its scatter mode.  Each translation unit instantiates the mode it launches.
#pragma once
#include <cooperative_groups.h>

#include <algorithm>
#include <mutex>

#include "bjx_handle.h"

namespace bjx {

// Eigensolver (k_lrd_eig): the top-k by |lam - 1| of R span the dominant-|mu| invariant subspace of A = R - I.  One
// cluster of 8 CTAs holds A row-partitioned in shared memory (D <= 512: at most 64 rows of 513 floats per CTA) and runs
// block orthogonal iteration with b = min(D, 2k + 16) columns: Y = A V, with V read slice by slice from the other CTAs
// through distributed shared memory; V = orth(Y) by CholeskyQR2 (the b x b Gram matrix reduced across the cluster in
// rank order, Cholesky and the triangular inverse in float64 by one warp); Rayleigh-Ritz at the first iteration and every
// kEigRR-th: T = V^T A V, cyclic Jacobi (float64, round-robin ordering, one CTA -- every CTA runs the same one, so all
// agree without a broadcast), V <- V W.  It stops when every selected Ritz pair has ||A u - mu u|| <= 1e-5 max|mu|, or
// at kEigMaxIter iterations, which sets the sticky non-converged flag.  The next step warm-starts from the stored Ritz
// basis; the first starts from a fixed pseudo-random basis.  With D <= b, V spans everything and the first Rayleigh-Ritz
// is the full Jacobi eigh of A.  Every reduction has a fixed order: two runs are bit-identical.
enum { LRD_ENGAGED = 0, LRD_ITERS, LRD_RESID, LRD_NOCONV, LRD_ITERS_SUM, LRD_ITERS_MAX, LRD_SOLVES, LRD_WARM };
constexpr int kLrdHdr = 16;
constexpr int kLrdMaxDim = 512, kLrdMaxRank = 16;
constexpr int kEigCtas = 8, kEigThreads = 512, kEigB = 48, kEigMaxIter = 300, kEigRR = 4, kJacobiSweeps = 30;
constexpr float kEigTol = 1e-5f, kLamFloor = 1e-6f;

inline int lrd_basis_cols(int D, int k) { return std::min(D, 2 * k + 16); }

__device__ __forceinline__ double warp_sum_d(double v) {
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

__device__ __forceinline__ float lrd_floor(float l) { return isnan(l) ? l : fmaxf(l, kLamFloor); }  // jnp.maximum keeps NaN
__device__ __forceinline__ float eig_hash(uint32_t i, uint32_t j) {  // cold-start basis entry in [-1, 1)
  uint32_t x = (i * 0x9E3779B1u) ^ ((j + 0x7F4A7C15u) * 0x85EBCA77u);
  x ^= x >> 16; x *= 0x7FEB352Du; x ^= x >> 15; x *= 0x846CA68Bu; x ^= x >> 16;
  return (float)(x >> 8) * (2.0f / 16777216.0f) - 1.0f;
}

static size_t eig_rows(int D) { return (size_t)(D + kEigCtas - 1) / kEigCtas; }
__host__ __device__ inline size_t round4(size_t n) { return (n + 3) & ~(size_t)3; }
static size_t eig_smem_bytes(int D) {
  const size_t RW = eig_rows(D);
  return (3 * kEigB * kEigB + 2 * kEigB) * sizeof(double) + (kEigB + 16) * sizeof(int) +
         (round4(D) + round4(RW * (D + 1)) + 3 * RW * kEigB) * sizeof(float);
}

namespace cg = cooperative_groups;

// the eigensolver (see above).  gate && n >= 2 D of the merged accumulator, else nothing.  cm: n, mean; W: merged
// covariance [D, D].  Writes sigma, U (top k by |mu|, descending), lam (floored), the Ritz basis and the diagnostics.
// kScatter (the low-rank window adaptation, bjx_lowrank_window.cu): W is already the symmetric matrix to solve -- no
// correlation, shift 0, no gate -- the top k are selected by the largest eigenvalue, lam gets the raw eigenvalues and
// sigma and cm are not read.  kScatter = false is the MEADS-LRD solve, compiled from the same code as before.
template <bool kScatter>
__global__ void __cluster_dims__(kEigCtas, 1, 1) __launch_bounds__(kEigThreads)
    k_lrd_eig(int D, int k, int B, int gate, const float* __restrict__ cm, const float* __restrict__ W,
              float* __restrict__ hdr, float* __restrict__ sigma, float* __restrict__ U, float* __restrict__ lam,
              float* __restrict__ basis) {
  if constexpr (!kScatter) {
    if (!(gate && cm[0] >= 2.f * (float)D)) return;
  }
  extern __shared__ __align__(16) unsigned char eig_smem[];
  constexpr int NB = kEigB, NT = kEigThreads;
  cg::cluster_group cl = cg::this_cluster();
  const int rank = (int)cl.block_rank(), tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int RW = (D + kEigCtas - 1) / kEigCtas, r0 = rank * RW, nr = max(0, min(RW, D - r0)), lda = D + 1;
  double* Gp = reinterpret_cast<double*>(eig_smem);  // this CTA's partial of a cluster reduction (read remotely)
  double* G = Gp + NB * NB;                          // the reduced matrix (Cholesky factor in place)
  double* Wm = G + NB * NB;                          // Jacobi eigenvectors / triangular inverse
  double* theta = Wm + NB * NB;
  double* cs = theta + NB;                           // Jacobi rotations of one round: c[24] | s[24]
  int* order = reinterpret_cast<int*>(cs + NB);
  int* flag = order + NB;                            // [0] Jacobi converged, [1] eigenpairs converged
  float* sig = reinterpret_cast<float*>(flag + 16);
  float* A = sig + round4(D);
  float* V = A + round4((size_t)RW * lda);
  float* Y = V + RW * NB;
  float* buf = Y + RW * NB;
  const bool warm = hdr[LRD_WARM] != 0.f;

  if constexpr (kScatter) {
    for (int e = tid; e < nr * D; e += NT) {
      const int i = e / D, j = e - i * D;
      A[i * lda + j] = W[(size_t)(r0 + i) * D + j];
    }
  } else {
    // correlation (metric_estimators.py:599-605) minus the identity, this CTA's rows
    for (int d = tid; d < D; d += NT) {
      const float s = sqrtf(fmaxf(W[(size_t)d * D + d], 0.f));
      sig[d] = s <= 0.f ? 1.f : s;
    }
    __syncthreads();
    for (int e = tid; e < nr * D; e += NT) {
      const int i = e / D, j = e - i * D, gi = r0 + i;
      const float r = W[(size_t)gi * D + j] * (1.f / sig[gi]) * (1.f / sig[j]);
      A[i * lda + j] = gi == j ? r - 1.f : r;
    }
  }
  for (int e = tid; e < RW * NB; e += NT) {
    const int i = e / NB, j = e - i * NB;
    Y[e] = (i < nr && j < B) ? (warm ? basis[(size_t)(r0 + i) * B + j] : eig_hash(r0 + i, j)) : 0.f;
  }
  __syncthreads();

  // G[0, n) = sum over the cluster's CTAs (rank order) of Gp[0, n)
  auto cluster_sum = [&](int n) {
    cl.sync();
    for (int e = tid; e < n; e += NT) {
      double s = 0.0;
      for (int r = 0; r < kEigCtas; ++r) s += cl.map_shared_rank(Gp, r)[e];
      G[e] = s;
    }
    cl.sync();
  };
  // Gp[i, j] = sum over this CTA's rows of X[row, i] Z[row, j]
  auto gram = [&](const float* X, const float* Z) {
    for (int e = tid; e < NB * NB; e += NT) {
      const int i = e / NB, j = e - i * NB;
      double s = 0.0;
      if (i < B && j < B)
        for (int r = 0; r < nr; ++r) s = fma((double)X[r * NB + i], (double)Z[r * NB + j], s);
      Gp[e] = s;
    }
  };
  // dst = src M for the B x B matrix M (upper triangular when tri), this CTA's rows
  auto apply = [&](const float* src, const double* M, bool tri, float* dst) {
    for (int e = tid; e < RW * NB; e += NT) {
      const int r = e / NB, j = e - r * NB;
      double s = 0.0;
      if (r < nr && j < B)
        for (int i = 0; i <= (tri ? j : B - 1); ++i) s = fma((double)src[r * NB + i], M[i * NB + j], s);
      dst[e] = (float)s;
    }
    __syncthreads();
  };
  // dst = src R^-1 with src^T src = R^T R over the cluster (one CholeskyQR pass); src and dst are distinct
  auto orth = [&](const float* src, float* dst) {
    gram(src, src);
    cluster_sum(NB * NB);
    if (warp == 0) {
      double mx = 0.0;
      for (int i = 0; i < B; ++i) mx = fmax(mx, G[i * NB + i]);
      if (mx > 0.0) {
        const double fl = 1e-15 * mx;  // keeps a (numerically) dependent column finite; the second pass restores it
        for (int j = 0; j < B; ++j) {
          double s0 = 0.0, s1 = 0.0;
          const int i0 = lane, i1 = lane + 32;
          if (i0 >= j && i0 < B) {
            s0 = G[j * NB + i0];
            for (int t = 0; t < j; ++t) s0 -= G[t * NB + j] * G[t * NB + i0];
          }
          if (i1 >= j && i1 < B) {
            s1 = G[j * NB + i1];
            for (int t = 0; t < j; ++t) s1 -= G[t * NB + j] * G[t * NB + i1];
          }
          const double piv = __shfl_sync(0xffffffffu, (j >> 5) ? s1 : s0, j & 31);
          const double rjj = sqrt(fmax(piv, fl));
          __syncwarp();
          if (i0 >= j && i0 < B) G[j * NB + i0] = i0 == j ? rjj : s0 / rjj;
          if (i1 >= j && i1 < B) G[j * NB + i1] = i1 == j ? rjj : s1 / rjj;
          __syncwarp();
        }
        for (int c = lane; c < B; c += 32)  // column c of R^-1 by back substitution
          for (int i = B - 1; i >= 0; --i) {
            double x = i == c ? 1.0 : 0.0;
            if (i < c)
              for (int t = i + 1; t <= c; ++t) x -= G[i * NB + t] * Wm[t * NB + c];
            Wm[i * NB + c] = i <= c ? x / G[i * NB + i] : 0.0;
          }
      } else {  // A V = 0 (or NaN): keep the basis
        for (int e = lane; e < NB * NB; e += 32) Wm[e] = (e / NB == e % NB) ? 1.0 : 0.0;
      }
    }
    __syncthreads();
    apply(src, Wm, true, dst);
  };
  // Y = A V; V is gathered slice by slice from every CTA through distributed shared memory
  auto matmul = [&]() {
    cl.sync();
    const int rp = tid >> 4, cq = tid & 15;  // rows 2 rp, 2 rp + 1; columns 3 cq .. 3 cq + 2
    float acc[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
    for (int s = 0; s < kEigCtas; ++s) {
      const int ns = max(0, min(RW, D - s * RW));
      if (ns == 0) break;
      const float4* src = reinterpret_cast<const float4*>(cl.map_shared_rank(V, s));
      float4* dst = reinterpret_cast<float4*>(buf);
      for (int e = tid; e < ns * (NB / 4); e += NT) dst[e] = src[e];
      __syncthreads();
      // rows past this CTA's RW are not stored: their threads read row RW - 1 and discard the result
      const float* a0 = A + min(2 * rp, RW - 1) * lda + s * RW;
      const float* a1 = A + min(2 * rp + 1, RW - 1) * lda + s * RW;
      const float* b = buf + 3 * cq;
      for (int jj = 0; jj < ns; ++jj) {
        const float x0 = a0[jj], x1 = a1[jj];
        const float b0 = b[jj * NB], b1 = b[jj * NB + 1], b2 = b[jj * NB + 2];
        acc[0][0] = fmaf(x0, b0, acc[0][0]); acc[0][1] = fmaf(x0, b1, acc[0][1]); acc[0][2] = fmaf(x0, b2, acc[0][2]);
        acc[1][0] = fmaf(x1, b0, acc[1][0]); acc[1][1] = fmaf(x1, b1, acc[1][1]); acc[1][2] = fmaf(x1, b2, acc[1][2]);
      }
      __syncthreads();
    }
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c)
        if (2 * rp + r < RW) Y[(2 * rp + r) * NB + 3 * cq + c] = (2 * rp + r < nr) ? acc[r][c] : 0.f;
    __syncthreads();
  };
  // cyclic Jacobi on the symmetric Gp (order n2 = B rounded up to even, padded with zeros): eigenvalues to theta,
  // eigenvectors to Wm.  Round-robin pairing, n2 / 2 disjoint rotations per round.
  auto jacobi = [&]() {
    const int n2 = B + (B & 1), half = n2 / 2;
    double* M = Gp;
    for (int e = tid; e < NB * NB; e += NT) {
      const int i = e / NB, j = e - i * NB;
      Wm[e] = i == j ? 1.0 : 0.0;
      if (i >= B || j >= B) M[e] = 0.0;
    }
    __syncthreads();
    auto pair_of = [&](int m, int rd, int& p, int& q) {
      if (m == 0) { p = rd % (n2 - 1); q = n2 - 1; }
      else { p = (rd + m) % (n2 - 1); q = (rd - m + n2 - 1) % (n2 - 1); }
    };
    for (int sweep = 0; sweep < kJacobiSweeps; ++sweep) {
      for (int rd = 0; rd < n2 - 1; ++rd) {
        if (tid < half) {
          int p, q;
          pair_of(tid, rd, p, q);
          const double app = M[p * NB + p], aqq = M[q * NB + q], apq = M[p * NB + q];
          double c = 1.0, s = 0.0;
          if (apq != 0.0) {
            const double tau = (aqq - app) / (2.0 * apq);
            const double t = (tau >= 0.0 ? 1.0 : -1.0) / (fabs(tau) + sqrt(1.0 + tau * tau));
            c = 1.0 / sqrt(1.0 + t * t);
            s = t * c;
          }
          cs[tid] = c;
          cs[24 + tid] = s;
        }
        __syncthreads();
        for (int e = tid; e < half * n2; e += NT) {  // rows p, q <- J^T rows
          const int m = e / n2, col = e - m * n2;
          int p, q;
          pair_of(m, rd, p, q);
          const double c = cs[m], s = cs[24 + m], x = M[p * NB + col], y = M[q * NB + col];
          M[p * NB + col] = c * x - s * y;
          M[q * NB + col] = s * x + c * y;
        }
        __syncthreads();
        for (int e = tid; e < half * n2; e += NT) {  // columns p, q <- columns J, also for the eigenvectors
          const int m = e / n2, row = e - m * n2;
          int p, q;
          pair_of(m, rd, p, q);
          const double c = cs[m], s = cs[24 + m];
          double x = M[row * NB + p], y = M[row * NB + q];
          M[row * NB + p] = c * x - s * y;
          M[row * NB + q] = s * x + c * y;
          x = Wm[row * NB + p]; y = Wm[row * NB + q];
          Wm[row * NB + p] = c * x - s * y;
          Wm[row * NB + q] = s * x + c * y;
        }
        __syncthreads();
      }
      if (warp == 0) {
        double off = 0.0, tot = 0.0;
        for (int e = lane; e < n2 * n2; e += 32) {
          const int i = e / n2, j = e - i * n2;
          const double v = M[i * NB + j] * M[i * NB + j];
          tot += v;
          if (i != j) off += v;
        }
        off = warp_sum_d(off);
        tot = warp_sum_d(tot);
        if (lane == 0) flag[0] = off <= 1e-28 * tot ? 1 : 0;
      }
      __syncthreads();
      const bool done = flag[0];
      __syncthreads();
      if (done) break;
    }
    for (int j = tid; j < B; j += NT) theta[j] = M[j * NB + j];
    __syncthreads();
  };

  orth(Y, V);
  orth(V, Y);
  { float* t = V; V = Y; Y = t; }
  int it = 0;
  bool converged = false;
  double resid = 0.0;
  while (true) {
    ++it;
    matmul();
    if (it == 1 || it % kEigRR == 0 || it == kEigMaxIter) {  // Rayleigh-Ritz and the residuals of the selected pairs
      gram(V, Y);
      cluster_sum(NB * NB);
      for (int e = tid; e < NB * NB; e += NT) {
        const int i = e / NB, j = e - i * NB;
        Gp[e] = 0.5 * (G[i * NB + j] + G[j * NB + i]);
      }
      __syncthreads();
      jacobi();
      apply(V, Wm, false, buf);
      for (int e = tid; e < RW * NB; e += NT) V[e] = buf[e];
      __syncthreads();
      apply(Y, Wm, false, buf);
      for (int e = tid; e < RW * NB; e += NT) Y[e] = buf[e];
      if (tid == 0) {  // scores |lam - 1| of the float32 eigenvalues it returns, descending; ties: the larger lam first
        for (int j = 0; j < B; ++j) order[j] = j;  // (argsort(scores)[::-1] over eigh's ascending eigenvalues)
        if constexpr (kScatter) {  // the largest eigenvalues, descending
          for (int m = 0; m < B; ++m) {
            int best = m;
            for (int j = m + 1; j < B; ++j)
              if (theta[order[j]] > theta[order[best]]) best = j;
            const int t = order[m]; order[m] = order[best]; order[best] = t;
          }
        } else {
          auto lam_f = [&](int j) { return (float)theta[j] + 1.0f; };
          for (int m = 0; m < B; ++m) {
            int best = m;
            for (int j = m + 1; j < B; ++j) {
              const float lj = lam_f(order[j]), lb = lam_f(order[best]);
              const float a = fabsf(lj - 1.0f), b = fabsf(lb - 1.0f);
              if (a > b || (a == b && lj > lb)) best = j;
            }
            const int t = order[m]; order[m] = order[best]; order[best] = t;
          }
        }
      }
      __syncthreads();
      if (warp < k) {
        const int j = order[warp];
        const double th = theta[j];
        double s = 0.0;
        for (int r = lane; r < nr; r += 32) {
          const double v = (double)Y[r * NB + j] - th * (double)V[r * NB + j];
          s = fma(v, v, s);
        }
        s = warp_sum_d(s);
        if (lane == 0) Gp[warp] = s;
      }
      cluster_sum(k);
      if (tid == 0) {
        const double mx = fabs(theta[order[0]]);
        double rmax = 0.0;
        for (int m = 0; m < k; ++m) rmax = fmax(rmax, sqrt(G[m]));
        flag[1] = rmax <= (double)kEigTol * mx ? 1 : 0;
        cs[0] = mx > 0.0 ? rmax / mx : rmax;  // cs is free between Jacobi calls: it hands the residual to every thread
      }
      __syncthreads();
      converged = flag[1] != 0;
      resid = cs[0];
      __syncthreads();
      if (converged || it == kEigMaxIter) break;
    }
    orth(Y, V);
    orth(V, Y);
    { float* t = V; V = Y; Y = t; }
  }
  for (int e = tid; e < nr * k; e += NT) {
    const int i = e / k, m = e - i * k;
    U[(size_t)(r0 + i) * k + m] = V[i * NB + order[m]];
  }
  for (int e = tid; e < nr * B; e += NT) {
    const int i = e / B, j = e - i * B;
    basis[(size_t)(r0 + i) * B + j] = V[i * NB + j];
  }
  if (rank == 0) {
    if constexpr (kScatter) {
      for (int m = tid; m < k; m += NT) lam[m] = (float)theta[order[m]];
    } else {
      for (int d = tid; d < D; d += NT) sigma[d] = sig[d];
      for (int m = tid; m < k; m += NT) lam[m] = lrd_floor((float)theta[order[m]] + 1.0f);
    }
    if (tid == 0) {
      hdr[LRD_ITERS] = (float)it;
      hdr[LRD_RESID] = (float)resid;
      if (!converged) hdr[LRD_NOCONV] = 1.f;
      hdr[LRD_ITERS_SUM] += (float)it;
      hdr[LRD_ITERS_MAX] = fmaxf(hdr[LRD_ITERS_MAX], (float)it);
      hdr[LRD_SOLVES] += 1.f;
      hdr[LRD_WARM] = 1.f;
    }
  }
  cl.sync();  // no CTA leaves while another may still read its shared memory
}

// the shared-memory opt-in of one instance of k_lrd_eig, once per device, at the size of the largest dimension
template <bool kScatter>
inline int eig_smem_opt_in(bjx_handle_t h) {
  static std::mutex mu;
  static bool done[64] = {};
  std::lock_guard<std::mutex> lock(mu);
  const int dev = h->cfg.device;
  if (dev < 0 || dev >= 64 || !done[dev]) {
    BJX_CUDA(cudaFuncSetAttribute(k_lrd_eig<kScatter>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)eig_smem_bytes(kLrdMaxDim)));
    if (dev >= 0 && dev < 64) done[dev] = true;
  }
  return 0;
}

}  // namespace bjx
