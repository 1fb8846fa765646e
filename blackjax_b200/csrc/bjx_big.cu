// Large rows (1024 < D <= 18432, D % 4 == 0): one CTA owns one chain and keeps the row in shared memory for the entire
// launch -- the same "state never round-trips HBM between leapfrogs" design as the warp-per-chain kernels
// (bjx_kernels.cuh), for rows that no longer fit a warp's registers.  The kernels shared with the plug-ins of user-defined
// big-row targets (init, n-step leapfrog with the momentum in registers, the one-chain-per-CTA HMC transition) live in
// bjx_big.cuh; this file holds the target-independent kernels (momentum draw, energy), the host dispatch, and BASELINE
// config 5's transition kernel: the hierarchical logistic regression (D = 10000) with TWO chains per CTA
// (k_big2_hmc_hier), bound by the 8 G sigmoid evaluations per leapfrog (MUFU pipe 56 %, issue slots 66 %), not by HBM.
//
// Same reference functions as the warp kernels: hmc.py:90-92 (init), metrics.py:260-270 (momentum draw,
// kinetic energy), integrators.py:104-150 (velocity Verlet), hmc.py:279-312 (transition),
// proposal.py:45-48,214-235 (accept).  Diagonal metrics only; NUTS is not built for this size class.
#include "bjx_handle.h"
#include "bjx_internal.h"
#include "bjx_big.cuh"
#include "bjx_prng.cuh"

using namespace bjx;

namespace bjx {
__global__ void __launch_bounds__(kBigThreads) k_big_momentum(BigParams P, const uint32_t* __restrict__ keys,
                                                              float* __restrict__ p_out) {
  const int c = blockIdx.x;
  const Key k = P.key_shared ? fold_in(Key{keys[0], keys[1]}, P.chain_offset + (uint32_t)c) : Key{keys[2 * c], keys[2 * c + 1]};
  const float* ms = P.msqrt + (size_t)c * P.imm_stride;
  for (int i = threadIdx.x; i < P.D; i += kBigThreads) p_out[(size_t)c * P.D + i] = __ldg(ms + i) * normal_at(k, (uint32_t)i);
}

__global__ void __launch_bounds__(kBigThreads) k_big_energy(BigParams P, const float* __restrict__ p_in,
                                                            const float* __restrict__ logp, float* __restrict__ e) {
  __shared__ float red[kBigWarps];
  const int c = blockIdx.x;
  const float* imm = P.imm + (size_t)c * P.imm_stride;
  float acc[1] = {0.f};
  for (int i = threadIdx.x; i < P.D; i += kBigThreads) {
    const float pv = p_in[(size_t)c * P.D + i];
    acc[0] = fmaf(__ldg(imm + i) * pv, pv, acc[0]);
  }
  block_sum<1>(acc, red);
  if (threadIdx.x == 0) e[c] = -logp[c] + 0.5f * acc[0];
}

// ---------------------------------------------------------------------------------------------------------------------
// Hierarchical logistic regression, TWO chains per CTA (BASELINE config 5's transition kernel).
//
// k_big_hmc above spends its time on the 8 G observations of a gradient evaluation, and every CTA streams the same 640 KB
// of covariates through L2 -> SM once per leapfrog step (419 GB per 32768-chain transition: half of the L2 throughput
// cap, with every consuming FMA waiting on it).  Here a CTA advances two chains together: a thread loads the covariates
// of a group ONCE and evaluates the group for both chains (half the L2 traffic and load / index instructions per chain,
// twice the independent work behind every load).  To fit two rows per SM the ownership is aligned: thread t owns elements
// i = t + T k of both rows AND the groups i - 4 that produce those gradient elements, so q, p and grad of the group
// intercepts are thread-private -- p lives in registers, q and grad in shared memory (2 x 2 x 40 KB) that only the owner
// touches, and no barrier orders the row passes.  Only the four hyper-parameters (elements 0..3) are shared: one barrier
// after the position update, and the block reduction of the 5 + 5 sums.
// Measured at 32768 x 10000, L = 20 (scripts/bench_c5.py): one chain per CTA 65.0 ms; this kernel with 768 threads (80
// registers) 55.2 ms, 640 threads 48.0 ms, 512 threads (128 registers: nothing spills) 41.8 ms, 384 threads 49.2 ms; with
// the next group's covariates prefetched into a second register set 47.8 ms (512 threads) -- two chains already put 16
// independent observations behind every load, the extra registers cost more than the prefetch hides.
template <int T>
__device__ __forceinline__ void block_sum2(float (&v)[10], float* red /*[10 * T/32]*/) {
  constexpr int W = T / 32;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 10; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
  }
  __syncthreads();  // protect red from the previous use
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < 10; ++k) red[k * W + wid] = v[k];
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 10; ++k) {  // every warp reduces the W partials with the same shuffle tree: identical on all threads
    float s = (lane < W) ? red[k * W + lane] : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    v[k] = s;
  }
}

template <int T, bool WANT_LOGP>
__device__ __forceinline__ void hier2_value_and_grad(const BigParams& P, const float* q0, const float* q1, float* g0, float* g1,
                                                     float* red, float (&logp)[2]) {
  const int tid = threadIdx.x, D = P.D;
  const float* qs[2] = {q0, q1};
  float* gs[2] = {g0, g1};
  float mu[2], lt[2], b0[2], b1[2], e2[2];
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    mu[c] = qs[c][0]; lt[c] = qs[c][1]; b0[c] = qs[c][2]; b1[c] = qs[c][3];
    e2[c] = expf(-2.0f * lt[c]);
  }
  float acc[10];  // per chain: ll, sum d, sum d^2, grad b0, grad b1
#pragma unroll
  for (int k = 0; k < 10; ++k) acc[k] = 0.f;
  for (int i = tid + (tid < 4 ? T : 0); i < D; i += T) {
    const int gidx = i - 4;
    const float4* xr = reinterpret_cast<const float4*>(P.data_x + (size_t)gidx * 16);
    float4 xv4[4];
#pragma unroll
    for (int k2 = 0; k2 < 4; ++k2) xv4[k2] = __ldg(xr + k2);
    const unsigned bits = __ldg(P.data_y + gidx);
    float alpha[2], ga[2] = {0.f, 0.f};
    alpha[0] = q0[i];
    alpha[1] = q1[i];
#pragma unroll
    for (int k2 = 0; k2 < 4; ++k2) {
      const float4 xv = xv4[k2];
      const float xs[2][2] = {{xv.x, xv.y}, {xv.z, xv.w}};
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const bool yb = (bits >> (2 * k2 + u)) & 1u;
#pragma unroll
        for (int c = 0; c < 2; ++c) {  // same arithmetic as big_value_and_grad (error bounds: tests/test_gpu_round2.py)
          const float eta = alpha[c] + b0[c] * xs[u][0] + b1[c] * xs[u][1];
          float ex, rc;
          asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(ex) : "f"(fabsf(eta) * -1.4426950408889634f));
          asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rc) : "f"(1.0f + ex));
          const float sig = (eta >= 0.f) ? rc : ex * rc;
          const float r = (yb ? 1.0f : 0.0f) - sig;
          if constexpr (WANT_LOGP) {
            float l2;
            asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(l2) : "f"(rc));
            const float softplus = fmaf(-0.69314718f, l2, fmaxf(eta, 0.f));
            acc[5 * c + 0] += (yb ? eta : 0.0f) - softplus;
          }
          ga[c] += r;
          acc[5 * c + 3] = fmaf(r, xs[u][0], acc[5 * c + 3]);
          acc[5 * c + 4] = fmaf(r, xs[u][1], acc[5 * c + 4]);
        }
      }
    }
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const float d = alpha[c] - mu[c];
      acc[5 * c + 1] += d;
      acc[5 * c + 2] = fmaf(d, d, acc[5 * c + 2]);
      gs[c][i] = -d * e2[c] + ga[c];
    }
  }
  block_sum2<T>(acc, red);
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    // elements 0..3 belong to threads 0..3
    if (tid == 0) gs[c][0] = -0.01f * mu[c] + e2[c] * acc[5 * c + 1];
    if (tid == 1) gs[c][1] = -lt[c] + e2[c] * acc[5 * c + 2] - (float)P.G;
    if (tid == 2) gs[c][2] = -0.16f * b0[c] + acc[5 * c + 3];
    if (tid == 3) gs[c][3] = -0.16f * b1[c] + acc[5 * c + 4];
    logp[c] = -0.005f * mu[c] * mu[c] - 0.5f * lt[c] * lt[c] - 0.08f * (b0[c] * b0[c] + b1[c] * b1[c]) +
              (-0.5f * e2[c] * acc[5 * c + 2] - (float)P.G * lt[c]) + acc[5 * c + 0] + P.logp_offset;
  }
}

// whole HMC transition (hmc.py:279-312) of chains 2b and 2b + 1
template <int T>
__global__ void __launch_bounds__(T) k_big2_hmc_hier(BigParams P, const uint32_t* __restrict__ keys, const float* q_in,
                                                     const float* logp_in, const float* g_in, float* q_out, float* logp_out,
                                                     float* g_out, int L, InfoPtrs info) {
  constexpr int NK = (10240 + T - 1) / T;  // elements per thread (rows up to 10240 dims)
  extern __shared__ __align__(16) float sm[];
  const int D = P.D, tid = threadIdx.x;
  float* qs[2] = {sm, sm + D};
  float* gs[2] = {sm + 2 * (size_t)D, sm + 3 * (size_t)D};
  float* red = sm + 4 * (size_t)D;
  int ch[2];
  bool live[2];
  ch[0] = 2 * blockIdx.x;
  ch[1] = min(2 * blockIdx.x + 1, P.C - 1);   // an odd chain count: the last CTA advances its chain twice, stores it once
  live[0] = true;
  live[1] = (2 * blockIdx.x + 1) < P.C;
  float p[2][NK];
  Key kint[2];
  float e0[2], logp0[2], eps[2];
  const float* imm[2];
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    const size_t ro = (size_t)ch[c] * D;
    const Key rng = P.key_shared ? fold_in(Key{keys[0], keys[1]}, P.chain_offset + (uint32_t)ch[c])
                                 : Key{keys[2 * ch[c]], keys[2 * ch[c] + 1]};
    const Key km = fold_in(rng, 0u);
    kint[c] = fold_in(rng, 1u);  // hmc.py:299
    imm[c] = P.imm + (size_t)ch[c] * P.imm_stride;
    const float* ms = P.msqrt + (size_t)ch[c] * P.imm_stride;
    float kin[10] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < NK; ++k) {
      const int i = tid + T * k;
      p[c][k] = 0.f;
      if (i < D) {
        qs[c][i] = __ldcs(q_in + ro + i);
        gs[c][i] = __ldcs(g_in + ro + i);
        const float pv = __ldg(ms + i) * normal_at(km, (uint32_t)i);  // hmc.py:302
        p[c][k] = pv;
        if (info.momentum && live[c]) info.momentum[ro + i] = pv;
        kin[0] = fmaf(__ldg(imm[c] + i) * pv, pv, kin[0]);
      }
    }
    block_sum2<T>(kin, red);
    logp0[c] = logp_in[ch[c]];
    e0[c] = -logp0[c] + 0.5f * kin[0];  // hmc.py:159
    eps[c] = P.eps_dev ? P.eps_dev[ch[c]] : P.eps;
  }
  float logp[2] = {logp0[0], logp0[1]};
  if (L > 0) {
    // velocity Verlet (integrators.py:104-150); between two steps the closing and the opening half kick share the pass
    auto kick_drift = [&](bool two_kicks) {
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const float eh = eps[c] * 0.5f, e1 = eps[c] * 1.0f;
#pragma unroll
        for (int k = 0; k < NK; ++k) {
          const int i = tid + T * k;
          if (i < D) {
            const float gv = gs[c][i];
            float pn = fmaf(eh, gv, p[c][k]);
            if (two_kicks) pn = fmaf(eh, gv, pn);
            p[c][k] = pn;
            qs[c][i] = fmaf(e1, __ldg(imm[c] + i) * pn, qs[c][i]);
          }
        }
      }
      __syncthreads();  // the hyper-parameters (elements 0..3) are read by every thread
    };
    kick_drift(false);
    for (int s = 0; s + 1 < L; ++s) {
      hier2_value_and_grad<T, false>(P, qs[0], qs[1], gs[0], gs[1], red, logp);
      kick_drift(true);
    }
    hier2_value_and_grad<T, true>(P, qs[0], qs[1], gs[0], gs[1], red, logp);
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const float eh = eps[c] * 0.5f;
#pragma unroll
      for (int k = 0; k < NK; ++k) {
        const int i = tid + T * k;
        if (i < D) p[c][k] = fmaf(eh, gs[c][i], p[c][k]);
      }
    }
  }
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    const size_t ro = (size_t)ch[c] * D;
    float kin[10] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < NK; ++k) {
      const int i = tid + T * k;
      if (i < D) kin[0] = fmaf(__ldg(imm[c] + i) * p[c][k], p[c][k], kin[0]);
    }
    block_sum2<T>(kin, red);
    const float e1 = -logp[c] + 0.5f * kin[0];  // hmc.py:160 (kinetic energy is even in p: the flip is implicit)
    float delta = e0[c] - e1;
    if (isnan(delta)) delta = -__int_as_float(0x7f800000);  // proposal.py:45-48
    const bool is_div = (-delta) > P.div_thr;
    float pa = expf(delta);
    pa = pa > 1.0f ? 1.0f : pa;                             // proposal.py:225
    const bool acc = uniform01(kint[c]) < pa;               // proposal.py:226
    if (!live[c]) continue;
#pragma unroll
    for (int k = 0; k < NK; ++k) {
      const int i = tid + T * k;
      if (i < D) {
        if (info.proposal_position) info.proposal_position[ro + i] = qs[c][i];
        if (info.proposal_momentum) info.proposal_momentum[ro + i] = -1.0f * p[c][k];  // hmc.py:158
        if (acc) {
          __stcs(q_out + ro + i, qs[c][i]);
          __stcs(g_out + ro + i, gs[c][i]);
        } else if (q_out != q_in) {
          __stcs(q_out + ro + i, __ldcs(q_in + ro + i));
          __stcs(g_out + ro + i, __ldcs(g_in + ro + i));
        }
      }
    }
    if (tid == 0) {
      if (acc || q_out != q_in) logp_out[ch[c]] = acc ? logp[c] : logp0[c];
      if (info.acceptance_rate) info.acceptance_rate[ch[c]] = pa;
      if (info.is_accepted) info.is_accepted[ch[c]] = acc;
      if (info.is_divergent) info.is_divergent[ch[c]] = is_div;
      if (info.energy) info.energy[ch[c]] = e1;
      if (info.num_integration_steps) info.num_integration_steps[ch[c]] = L;
    }
  }
}
}  // namespace bjx

static BigParams big_params(bjx_handle_t h, float eps, const float* eps_dev) {
  BigParams P;
  P.C = h->cfg.n_chains;
  P.D = h->cfg.dim;
  P.kind = h->cfg.target.kind;
  P.inv_var = h->cfg.target.inv_var;
  P.mean = h->cfg.target.mean;
  P.logp_offset = h->cfg.target.logp_offset;
  P.data_x = h->cfg.target.data_x;
  P.data_y = h->cfg.target.data_y;
  P.G = h->cfg.target.n_groups;
  P.user = h->cfg.target.user_params;
  P.n_user = h->cfg.target.n_user_params;
  P.imm = h->imm;
  P.imm_stride = (h->metric_kind == BJX_METRIC_DIAG_PER_CHAIN) ? h->cfg.dim : 0;
  P.msqrt = h->msqrt;
  P.eps = eps;
  P.eps_dev = eps_dev;
  P.div_thr = h->cfg.divergence_threshold;
  P.key_shared = h->key_shared;
  P.chain_offset = h->chain_offset;
  return P;
}

static int big_dispatch(bjx_handle_t h, int kernel_id, BigLaunchArgs& a) {
  a.stream = h->stream;
  int rc;
  switch (h->cfg.target.kind) {
    case BJX_TARGET_DIAG_GAUSSIAN: rc = big_launch<BJX_TARGET_DIAG_GAUSSIAN>(kernel_id, a); break;
    case BJX_TARGET_FUNNEL: rc = big_launch<BJX_TARGET_FUNNEL>(kernel_id, a); break;
    case BJX_TARGET_HIER_LOGIT: rc = big_launch<BJX_TARGET_HIER_LOGIT>(kernel_id, a); break;
    case BJX_TARGET_USER: {
      auto* pl = static_cast<bjx_plugin_s*>(h->cfg.target.user_plugin);
      if (!pl || !pl->launch_big)
        return bjx_fail(h, BJX_E_UNSUPPORTED, "this target plug-in was built for rows up to 1024 dims (no bjx_user::BigModel)");
      rc = pl->launch_big(kernel_id, &a);
      break;
    }
    default: return bjx_fail(h, BJX_E_UNSUPPORTED, "target not built for dim > 1024");
  }
  if (rc) return bjx_cuda_fail(h, (cudaError_t)rc, "big-row kernel launch");
  return 0;
}

int bjx_big_init_state(bjx_handle_t h, const float* q, float* logp_out, float* grad_out) {
  BigLaunchArgs a{};
  a.P = big_params(h, 0.f, nullptr);
  a.q_in = q; a.logp_out = logp_out; a.g_out = grad_out;
  return big_dispatch(h, BK_INIT, a);
}
int bjx_big_sample_momentum(bjx_handle_t h, const uint32_t* keys, float* p_out) {
  BigParams P = big_params(h, 0.f, nullptr);
  k_big_momentum<<<h->cfg.n_chains, kBigThreads, 0, h->stream>>>(P, keys, p_out);
  BJX_CHECK_LAUNCH("k_big_momentum");
  return 0;
}
int bjx_big_energy(bjx_handle_t h, const float* p, const float* logp, float* e_out) {
  BigParams P = big_params(h, 0.f, nullptr);
  k_big_energy<<<h->cfg.n_chains, kBigThreads, 0, h->stream>>>(P, p, logp, e_out);
  BJX_CHECK_LAUNCH("k_big_energy");
  return 0;
}
int bjx_big_leapfrog(bjx_handle_t h, float* q, float* p, float* logp, float* g, float eps, const float* eps_dev, int n) {
  BigLaunchArgs a{};
  a.P = big_params(h, eps, eps_dev);
  a.q_out = q; a.p_io = p; a.logp_out = logp; a.g_out = g; a.n = n;
  return big_dispatch(h, BK_LEAPFROG, a);
}
int bjx_big_hmc_step(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logp_in, const float* g_in,
                     float* q_out, float* logp_out, float* g_out, float eps, const float* eps_dev, int L,
                     const InfoPtrs& info) {
  BigParams P = big_params(h, eps, eps_dev);
  if (h->cfg.target.kind == BJX_TARGET_HIER_LOGIT && h->cfg.dim <= 10240) {
    // two chains per CTA, momentum in registers (see k_big2_hmc_hier); rows beyond 10240 run one chain per CTA
    const size_t smem = (4 * (size_t)h->cfg.dim + 10 * 32) * sizeof(float);
    const int ctas = (h->cfg.n_chains + 1) / 2;
    BJX_CUDA(cudaFuncSetAttribute(k_big2_hmc_hier<512>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_big2_hmc_hier<512><<<ctas, 512, smem, h->stream>>>(P, keys, q_in, logp_in, g_in, q_out, logp_out, g_out, L, info);
    BJX_CHECK_LAUNCH("k_big2_hmc_hier");
    return 0;
  }
  BigLaunchArgs a{};
  a.P = P;
  a.keys = keys; a.q_in = q_in; a.logp_in = logp_in; a.g_in = g_in;
  a.q_out = q_out; a.logp_out = logp_out; a.g_out = g_out; a.n = L; a.info = info;
  return big_dispatch(h, BK_HMC, a);
}
// MALA / Barker on the big rows: one transition (A.loop.step_keys == nullptr) or the native loop (bjx_langevin.cu)
int bjx_big_langevin(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logp_in, const float* g_in,
                     float* q_out, float* logp_out, float* g_out, float eps, const float* eps_dev, const LangevinArgs& A) {
  BigLaunchArgs a{};
  a.P = big_params(h, eps, eps_dev);
  a.keys = keys; a.q_in = q_in; a.logp_in = logp_in; a.g_in = g_in;
  a.q_out = q_out; a.logp_out = logp_out; a.g_out = g_out;
  a.langevin = A;
  return big_dispatch(h, BK_LANGEVIN, a);
}
// Elliptical slice sampling on the big rows: one transition (A.loop.step_keys == nullptr) or the native loop (bjx_ess.cu)
int bjx_big_ess(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logl_in, float* q_out,
                float* logl_out, const EssArgs& A) {
  BigLaunchArgs a{};
  a.P = big_params(h, 0.f, nullptr);
  a.keys = keys; a.q_in = q_in; a.logp_in = logl_in;
  a.q_out = q_out; a.logp_out = logl_out;
  a.ess = A;
  return big_dispatch(h, BK_ESS, a);
}
// Slice sampling on the big rows: one transition (A.loop.step_keys == nullptr) or the native loop (bjx_slice.cu)
int bjx_big_slice(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logp_in, float* q_out,
                  float* logp_out, float width, const float* width_dev, const SliceArgs& A) {
  BigLaunchArgs a{};
  a.P = big_params(h, width, width_dev);
  a.keys = keys; a.q_in = q_in; a.logp_in = logp_in;
  a.q_out = q_out; a.logp_out = logp_out;
  a.slice = A;
  return big_dispatch(h, BK_SLICE, a);
}
// Random-walk Metropolis on the big rows: one transition (A.loop.step_keys == nullptr) or the native loop (bjx_rw.cu)
int bjx_big_rw(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logp_in, float* q_out,
               float* logp_out, const RwArgs& A) {
  BigLaunchArgs a{};
  a.P = big_params(h, 0.f, nullptr);
  a.keys = keys; a.q_in = q_in; a.logp_in = logp_in;
  a.q_out = q_out; a.logp_out = logp_out;
  a.rw = A;
  return big_dispatch(h, BK_RW, a);
}
