// Kernels for rows beyond a warp (1024 < D <= 18432, D % 4 == 0): one CTA owns one chain (see bjx_big.cu for the design
// notes).  Header so that the plug-in of a user-defined target (bjx_plugin.cu with -DBJX_PLUGIN_BIG=1) instantiates the same
// kernels around the user's CTA-level value_and_grad (bjx_user::BigModel, include/bjx_user_target.h) as libbjx does around
// the built-in targets.
#pragma once
#include "../../include/bjx.h"
#include "bjx_kernels.cuh"
#include "bjx_launch.cuh"  // (LaunchArgs: part of the plug-in ABI number)

namespace bjx_user {
struct BigModel;  // defined by a big-row plug-in's source
}

namespace bjx {

constexpr int kBigThreads = 768;  // one CTA per SM (shared-memory bound): 24 warps hide the MUFU / L2 latency
constexpr int kBigWarps = kBigThreads / 32;

struct BigParams {
  int C, D;
  int kind;
  const float* inv_var;
  const float* mean;
  float logp_offset;
  const float* data_x;
  const uint8_t* data_y;
  int G;
  const float* user;   // BJX_TARGET_USER: the model's parameter block
  int n_user;
  const float* imm;
  long long imm_stride;
  const float* msqrt;
  float eps;
  const float* eps_dev;
  float div_thr;
  int key_shared;
  uint32_t chain_offset;
};

// block-wide sum of up to NV values per thread (result valid in all threads)
template <int NV>
__device__ __forceinline__ void block_sum(float (&v)[NV], float* red /*[NV*kBigWarps]*/) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
  }
  __syncthreads();  // protect red from the previous use
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < NV; ++k) red[k * kBigWarps + wid] = v[k];
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < kBigWarps; ++w) s += red[k * kBigWarps + w];
    v[k] = s;
  }
}

// value_and_grad of the target at the row q (shared memory) -> g (shared memory), returns logp (all threads).
// WANT_LOGP = false: only the gradient is consumed (interior steps of a fixed-length trajectory, where the value is
// dead -- as in the warp kernels); the hierarchical logistic model then skips the softplus (one MUFU of three and a
// quarter of the instructions per observation).
// CTA-level context of a user-defined big-row model (include/bjx_user_target.h)
struct BigUserCtx {
  const float* theta;  // parameter block [n_theta] (device memory, read-only)
  int n_theta;
  int D;
  int tid;             // threadIdx.x in [0, kBigThreads)
};
template <int TK>
struct BigUserOf { using type = void; };
template <>
struct BigUserOf<BJX_TARGET_USER> { using type = bjx_user::BigModel; };

template <int TK, bool WANT_LOGP = true>
__device__ __forceinline__ float big_value_and_grad(const BigParams& P, const float* q, float* g, float* red) {
  const int D = P.D, tid = threadIdx.x;
  if constexpr (TK == BJX_TARGET_USER) {
    const BigUserCtx u{P.user, P.n_user, D, tid};
    using M = typename BigUserOf<TK>::type;
    return M::template value_and_grad<WANT_LOGP>(u, q, g, red) + P.logp_offset;
  } else if constexpr (TK == BJX_TARGET_DIAG_GAUSSIAN) {
    float acc[1] = {0.f};
    for (int i = tid; i < D; i += kBigThreads) {
      const float d = P.mean ? q[i] - __ldg(P.mean + i) : q[i];
      const float t = d * -__ldg(P.inv_var + i);
      acc[0] = fmaf(d, t, acc[0]);
      g[i] = t;
    }
    if constexpr (!WANT_LOGP) return 0.f;
    block_sum<1>(acc, red);
    return 0.5f * acc[0] + P.logp_offset;
  } else if constexpr (TK == BJX_TARGET_FUNNEL) {
    const float y = q[0];
    float acc[1] = {0.f};
    for (int i = tid; i < D; i += kBigThreads) acc[0] = (i == 0) ? acc[0] : fmaf(q[i], q[i], acc[0]);
    block_sum<1>(acc, red);
    const float ss = acc[0], ey = expf(-y), n = (float)(D - 1), t = y / 3.0f;
    for (int i = tid; i < D; i += kBigThreads) g[i] = (i == 0) ? (-y / 9.0f + 0.5f * ey * ss - 0.5f * n) : -(ey * q[i]);
    return -0.5f * (t * t) + (-0.5f * ey * ss - 0.5f * n * y) + P.logp_offset;
  } else {  // BJX_TARGET_HIER_LOGIT
    const float mu = q[0], lt = q[1], b0 = q[2], b1 = q[3];
    const float e2 = expf(-2.0f * lt);
    float acc[5] = {0.f, 0.f, 0.f, 0.f, 0.f};  // ll, sum d, sum d^2, grad b0, grad b1
    // Software pipeline over this thread's groups, two register sets (A, B): the 64 bytes of covariates + the outcome byte
    // of the NEXT group are requested before the 8 observations of the current one are evaluated (the data is
    // L2-resident, ~1 us away; ncu before: half of the stall samples on the first FMA that consumes a covariate).
    auto load_group = [&](int gidx, float4 (&xv)[4], unsigned& bv, float& av) {
      if (gidx < P.G) {
        const float4* xr = reinterpret_cast<const float4*>(P.data_x + (size_t)gidx * 16);
#pragma unroll
        for (int k2 = 0; k2 < 4; ++k2) xv[k2] = __ldg(xr + k2);
        bv = __ldg(P.data_y + gidx);
        av = q[4 + gidx];
      }
    };
    auto eval_group = [&](int gidx, const float4 (&xv4)[4], unsigned bits, float alpha) {
      const float d = alpha - mu;
      float ga = 0.f;
#pragma unroll
      for (int k2 = 0; k2 < 4; ++k2) {
        const float4 xv = xv4[k2];  // (x_{2k2,0}, x_{2k2,1}, x_{2k2+1,0}, x_{2k2+1,1})
        const float xs[2][2] = {{xv.x, xv.y}, {xv.z, xv.w}};
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const bool yb = (bits >> (2 * k2 + u)) & 1u;
          const float eta = alpha + b0 * xs[u][0] + b1 * xs[u][1];
          // One exponential feeds both the sigmoid and the softplus, and the softplus reuses the sigmoid's reciprocal:
          //   ex = exp(-|eta|), r = 1 / (1 + ex), sigmoid = eta >= 0 ? r : ex r, softplus = max(eta, 0) - log(r).
          // ex2.approx / rcp.approx / lg2.approx: 3 MUFU + ~20 FP32/ALU instructions per observation (expf + an IEEE
          // division + log1pf + int-to-float conversions cost 70; __expf / __frcp_rn / (float)bit still 41, of which a
          // dozen guard subnormal ranges these arguments never reach).  Error bounds, checked against float64 in
          // tests/test_gpu_round2.py: |sigmoid error| <= 4e-7 (ex2 2 ulp, rcp 1 ulp), |softplus error| <= 3e-7 absolute.
          float ex, rc;
          asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(ex) : "f"(fabsf(eta) * -1.4426950408889634f));
          asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rc) : "f"(1.0f + ex));   // 1 + ex in [1, 2]
          const float sig = (eta >= 0.f) ? rc : ex * rc;
          const float r = (yb ? 1.0f : 0.0f) - sig;
          if constexpr (WANT_LOGP) {
            float l2;
            asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(l2) : "f"(rc));        // rc in [1/2, 1]
            const float softplus = fmaf(-0.69314718f, l2, fmaxf(eta, 0.f));
            acc[0] += (yb ? eta : 0.0f) - softplus;
          }
          ga += r;
          acc[3] = fmaf(r, xs[u][0], acc[3]);
          acc[4] = fmaf(r, xs[u][1], acc[4]);
        }
      }
      acc[1] += d;
      acc[2] = fmaf(d, d, acc[2]);
      g[4 + gidx] = -d * e2 + ga;
    };
    float4 xa[4], xb[4];
    unsigned ba = 0, bb = 0;
    float aa = 0.f, ab = 0.f;
    load_group(tid, xa, ba, aa);
    for (int gi = tid; gi < P.G; gi += 2 * kBigThreads) {
      load_group(gi + kBigThreads, xb, bb, ab);
      eval_group(gi, xa, ba, aa);
      load_group(gi + 2 * kBigThreads, xa, ba, aa);
      if (gi + kBigThreads < P.G) eval_group(gi + kBigThreads, xb, bb, ab);
    }
    block_sum<5>(acc, red);
    if (tid == 0) {
      g[0] = -0.01f * mu + e2 * acc[1];
      g[1] = -lt + e2 * acc[2] - (float)P.G;
      g[2] = -0.16f * b0 + acc[3];
      g[3] = -0.16f * b1 + acc[4];
    }
    return -0.005f * mu * mu - 0.5f * lt * lt - 0.08f * (b0 * b0 + b1 * b1) + (-0.5f * e2 * acc[2] - (float)P.G * lt) +
           acc[0] + P.logp_offset;
  }
}

__device__ __forceinline__ float big_kinetic(const BigParams& P, const float* imm, const float* p, float* red) {
  float acc[1] = {0.f};
  for (int i = threadIdx.x; i < P.D; i += kBigThreads) acc[0] = fmaf(__ldg(imm + i) * p[i], p[i], acc[0]);
  block_sum<1>(acc, red);
  return 0.5f * acc[0];
}

// n velocity-Verlet steps (integrators.py:104-150) on the row in shared memory; returns the log-density after the last
// one.  Between two steps the closing half kick of one and the opening half kick of the next run in the same pass over
// the row (two separately rounded FMAs, bit-identical to the step-by-step form), so an interior step is one pass +
// one gradient evaluation (gradient only: its log-density is dead) instead of two passes.
template <int TK>
__device__ __forceinline__ float big_trajectory(const BigParams& P, const float* imm, float* q, float* p, float* g,
                                                float eps, int n, float* red) {
  const float eh = eps * 0.5f, e1 = eps * 1.0f;
  if (n <= 0) return 0.f;
  for (int i = threadIdx.x; i < P.D; i += kBigThreads) {
    const float pn = fmaf(eh, g[i], p[i]);
    p[i] = pn;
    q[i] = fmaf(e1, __ldg(imm + i) * pn, q[i]);
  }
  __syncthreads();
  for (int s = 0; s + 1 < n; ++s) {
    big_value_and_grad<TK, false>(P, q, g, red);
    __syncthreads();
    for (int i = threadIdx.x; i < P.D; i += kBigThreads) {
      float pn = fmaf(eh, g[i], p[i]);   // second half kick of step s
      pn = fmaf(eh, g[i], pn);           // first half kick of step s + 1
      p[i] = pn;
      q[i] = fmaf(e1, __ldg(imm + i) * pn, q[i]);
    }
    __syncthreads();
  }
  const float logp = big_value_and_grad<TK, true>(P, q, g, red);
  __syncthreads();
  for (int i = threadIdx.x; i < P.D; i += kBigThreads) p[i] = fmaf(eh, g[i], p[i]);
  __syncthreads();
  return logp;
}

__device__ __forceinline__ void big_load(float* dst, const float* __restrict__ src, int D) {
  for (int i = threadIdx.x; i < D / 4; i += kBigThreads)
    reinterpret_cast<float4*>(dst)[i] = __ldcs(reinterpret_cast<const float4*>(src) + i);
}
__device__ __forceinline__ void big_store(float* __restrict__ dst, const float* src, int D) {
  for (int i = threadIdx.x; i < D / 4; i += kBigThreads)
    __stcs(reinterpret_cast<float4*>(dst) + i, reinterpret_cast<const float4*>(src)[i]);
}

template <int TK>
__global__ void __launch_bounds__(kBigThreads) k_big_init(BigParams P, const float* __restrict__ q_in,
                                                          float* __restrict__ logp_out, float* __restrict__ g_out) {
  extern __shared__ __align__(16) float sm[];
  float *q = sm, *g = sm + P.D, *red = sm + 2 * (size_t)P.D;
  const size_t ro = (size_t)blockIdx.x * P.D;
  big_load(q, q_in + ro, P.D);
  __syncthreads();
  const float logp = big_value_and_grad<TK>(P, q, g, red);
  __syncthreads();
  big_store(g_out + ro, g, P.D);
  if (threadIdx.x == 0) logp_out[blockIdx.x] = logp;
}

// n leapfrog steps per launch (bjx_leapfrog; n = 1 is the one-step kernel the HBM roofline is quoted on).  Thread t owns
// elements t + 768 k of the row, so the momentum is thread-private and stays in REGISTERS (NK per thread); only q and grad,
// which the target's value_and_grad addresses freely, live in shared memory: 2 x 4 D bytes instead of 3 x 4 D, and for
// rows up to 10752 dims two CTAs fit an SM, so one CTA's loads and stores overlap the other's arithmetic (with three rows
// and one CTA per SM the phases load -> compute -> store ran back to back: 0.45 of the HBM peak at 32768 x 10000).
template <int TK, int NK>
__global__ void __launch_bounds__(kBigThreads, (NK <= 14 && (TK == BJX_TARGET_DIAG_GAUSSIAN || TK == BJX_TARGET_FUNNEL)) ? 2 : 1)
    k_big_leapfrog(BigParams P, float* q_io, float* p_io, float* logp_io, float* g_io, int n_steps) {
  extern __shared__ __align__(16) float sm[];
  float *q = sm, *g = sm + P.D, *red = sm + 2 * (size_t)P.D;
  const int c = blockIdx.x, D = P.D, tid = threadIdx.x;
  const size_t ro = (size_t)c * D;
  const float* imm = P.imm + (size_t)c * P.imm_stride;
  const float eps = P.eps_dev ? P.eps_dev[c] : P.eps;
  const float eh = eps * 0.5f, e1 = eps * 1.0f;
  float p[NK];
  if (n_steps <= 0) return;
  // load + first half kick + position update in one pass (integrators.py:199-203,235-245)
#pragma unroll
  for (int k = 0; k < NK; ++k) {
    const int i = tid + kBigThreads * k;
    p[k] = 0.f;
    if (i < D) {
      const float pn = fmaf(eh, __ldcs(g_io + ro + i), __ldcs(p_io + ro + i));
      p[k] = pn;
      q[i] = fmaf(e1, __ldg(imm + i) * pn, __ldcs(q_io + ro + i));
    }
  }
  __syncthreads();
  for (int s = 0; s + 1 < n_steps; ++s) {
    big_value_and_grad<TK, false>(P, q, g, red);
    __syncthreads();
#pragma unroll
    for (int k = 0; k < NK; ++k) {
      const int i = tid + kBigThreads * k;
      if (i < D) {
        const float gv = g[i];
        float pn = fmaf(eh, gv, p[k]);   // second half kick of step s
        pn = fmaf(eh, gv, pn);           // first half kick of step s + 1
        p[k] = pn;
        q[i] = fmaf(e1, __ldg(imm + i) * pn, q[i]);
      }
    }
    __syncthreads();
  }
  const float logp = big_value_and_grad<TK, true>(P, q, g, red);
  __syncthreads();
#pragma unroll
  for (int k = 0; k < NK; ++k) {
    const int i = tid + kBigThreads * k;
    if (i < D) {
      const float gv = g[i];
      __stcs(p_io + ro + i, fmaf(eh, gv, p[k]));
      __stcs(g_io + ro + i, gv);
      __stcs(q_io + ro + i, q[i]);
    }
  }
  if (tid == 0) logp_io[c] = logp;
}

// whole HMC transition (hmc.py:279-312) with the row resident in shared memory
template <int TK>
__global__ void __launch_bounds__(kBigThreads) k_big_hmc(BigParams P, const uint32_t* __restrict__ keys, const float* q_in,
                                                         const float* logp_in, const float* g_in, float* q_out,
                                                         float* logp_out, float* g_out, int L, InfoPtrs info) {
  extern __shared__ __align__(16) float sm[];
  float *q = sm, *p = sm + P.D, *g = sm + 2 * (size_t)P.D, *red = sm + 3 * (size_t)P.D;
  const int c = blockIdx.x;
  const size_t ro = (size_t)c * P.D;
  big_load(q, q_in + ro, P.D);
  big_load(g, g_in + ro, P.D);
  const Key rng = P.key_shared ? fold_in(Key{keys[0], keys[1]}, P.chain_offset + (uint32_t)c) : Key{keys[2 * c], keys[2 * c + 1]};
  const Key km = fold_in(rng, 0u), ki = fold_in(rng, 1u);  // hmc.py:299
  const float* imm = P.imm + (size_t)c * P.imm_stride;
  const float* ms = P.msqrt + (size_t)c * P.imm_stride;
  for (int i = threadIdx.x; i < P.D; i += kBigThreads) {
    const float pv = __ldg(ms + i) * normal_at(km, (uint32_t)i);  // hmc.py:302
    p[i] = pv;
    if (info.momentum) info.momentum[ro + i] = pv;
  }
  __syncthreads();
  const float logp0 = logp_in[c];
  const float e0 = -logp0 + big_kinetic(P, imm, p, red);  // hmc.py:159
  const float eps = P.eps_dev ? P.eps_dev[c] : P.eps;
  const float logp = L > 0 ? big_trajectory<TK>(P, imm, q, p, g, eps, L, red) : logp0;  // trajectory.py:165
  const float e1 = -logp + big_kinetic(P, imm, p, red);  // hmc.py:160 (kinetic energy is even in p: the flip is implicit)
  float delta = e0 - e1;
  if (isnan(delta)) delta = -__int_as_float(0x7f800000);  // proposal.py:45-48
  const bool is_div = (-delta) > P.div_thr;
  float pa = expf(delta);
  pa = pa > 1.0f ? 1.0f : pa;                             // proposal.py:225
  const bool acc = uniform01(ki) < pa;                    // proposal.py:226
  if (info.proposal_position) big_store(info.proposal_position + ro, q, P.D);
  if (info.proposal_momentum)
    for (int i = threadIdx.x; i < P.D; i += kBigThreads) info.proposal_momentum[ro + i] = -1.0f * p[i];  // hmc.py:158
  if (acc) {
    big_store(q_out + ro, q, P.D);
    big_store(g_out + ro, g, P.D);
  } else if (q_out != q_in) {
    for (int i = threadIdx.x; i < P.D / 4; i += kBigThreads) {
      __stcs(reinterpret_cast<float4*>(q_out + ro) + i, __ldcs(reinterpret_cast<const float4*>(q_in + ro) + i));
      __stcs(reinterpret_cast<float4*>(g_out + ro) + i, __ldcs(reinterpret_cast<const float4*>(g_in + ro) + i));
    }
  }
  if (threadIdx.x == 0) {
    if (acc || q_out != q_in) logp_out[c] = acc ? logp : logp0;
    if (info.acceptance_rate) info.acceptance_rate[c] = pa;
    if (info.is_accepted) info.is_accepted[c] = acc;
    if (info.is_divergent) info.is_divergent[c] = is_div;
    if (info.energy) info.energy[c] = e1;
    if (info.num_integration_steps) info.num_integration_steps[c] = L;
  }
}

// MALA / Barker transitions (the warp kernels' langevin_transition_row, bjx_kernels.cuh) with a diagonal metric.  The
// position and the proposal's (y, grad y), which the target addresses freely, sit in shared memory; the gradient at the
// position is read from its [C, D] array where thread t uses elements t + 768 k (three rows fill the shared memory at
// 18432 dims, and a fourth in registers spills).  One launch runs one transition (A.loop.step_keys == nullptr: keys and
// A.info as bjx_hmc_step's) or the A.loop.num_steps transitions of the native loop, in place, with the position on chip
// throughout and the gradient row rewritten on acceptance.
template <int TK, int KIND>
__global__ void __launch_bounds__(kBigThreads) k_big_langevin(BigParams P, const uint32_t* __restrict__ keys,
                                                              const float* q_in, const float* logp_in, const float* g_in,
                                                              float* q_out, float* logp_out, float* g_out, LangevinArgs A) {
  extern __shared__ __align__(16) float sm[];
  float *xs = sm, *y = sm + P.D, *gy = sm + 2 * (size_t)P.D, *red = sm + 3 * (size_t)P.D;
  const int c = blockIdx.x, D = P.D, tid = threadIdx.x;
  const size_t ro = (size_t)c * D;
  __shared__ float langevin_slot[2];
  const LangevinScalars sc = langevin_scalars(P.eps_dev ? P.eps_dev[c] : P.eps, langevin_slot,
                                              KIND == LANGEVIN_MALA && tid == 0);
  const float eps = sc.eps;
  const float* ms = P.msqrt + (size_t)c * P.imm_stride;
  const float* imm = P.imm + (size_t)c * P.imm_stride;
  const bool loop = A.loop.step_keys != nullptr;
  const int T = loop ? A.loop.num_steps : 1;
  const float* gx = g_in + ro;  // the native loop: g_in == g_out, updated on acceptance
  big_load(xs, q_in + ro, D);
  float logp_x = logp_in[c];
  bool acc = false;
  __syncthreads();
  for (int t = 0; t < T; ++t) {
    // the transition's key, derived where each use needs it so that no key stays live across the target's evaluation
    auto rng = [&]() {
      const uint32_t* kt = loop ? A.loop.step_keys + 2 * t : keys;
      return P.key_shared ? fold_in(Key{kt[0], kt[1]}, P.chain_offset + (uint32_t)c) : Key{kt[2 * c], kt[2 * c + 1]};
    };
    float la, logp_y;  // log_p_accept; the proposal's log-density (the same in every thread)
    if constexpr (KIND == LANGEVIN_MALA) {
      const Key key_noise = fold_in(rng(), 0u);
      for (int i = tid; i < D; i += kBigThreads)
        y[i] = __fadd_rn(__fadd_rn(xs[i], __fmul_rn(eps, gx[i])), __fmul_rn(sc.s2(), normal_at(key_noise, (uint32_t)i)));
      __syncthreads();
      logp_y = big_value_and_grad<TK>(P, y, gy, red);
      __syncthreads();
      float sums[2] = {0.f, 0.f};
      for (int i = tid; i < D; i += kBigThreads) {
        const float tn = __fsub_rn(__fsub_rn(xs[i], y[i]), __fmul_rn(eps, gy[i]));
        const float tp = __fsub_rn(__fsub_rn(y[i], xs[i]), __fmul_rn(eps, gx[i]));
        sums[0] = __fmaf_rn(tn, tn, sums[0]);
        sums[1] = __fmaf_rn(tp, tp, sums[1]);
      }
      block_sum<2>(sums, red);
      la = safe_energy_diff(__fadd_rn(-logp_x, __fmul_rn(sc.w(), sums[1])), __fadd_rn(-logp_y, __fmul_rn(sc.w(), sums[0])));
    } else {
      const Key k0 = fold_in(rng(), 0u), key_normal = fold_in(k0, 0u), key_sign = fold_in(fold_in(k0, 1u), 0u);
      for (int i = tid; i < D; i += kBigThreads) {
        const float m = __ldg(ms + i);
        const float z = __fmul_rn(eps, normal_at(key_normal, (uint32_t)i));
        const float pb = expf(-log1pexp_naive(__fmul_rn(-__fmul_rn(m, gx[i]), z)));
        const float bz = uniform01(key_sign, (uint32_t)i) < pb ? z : -z;
        y[i] = __fadd_rn(xs[i], __fmul_rn(m, bz));
      }
      __syncthreads();
      logp_y = big_value_and_grad<TK>(P, y, gy, red);
      __syncthreads();
      float sums[4] = {0.f, 0.f, 0.f, 0.f};
      for (int i = tid; i < D; i += kBigThreads) {
        const float m = __ldg(ms + i), iv = __ldg(imm + i);
        const float d = __fsub_rn(xs[i], y[i]);
        const float v = __fmul_rn(iv, d), zt = __fmul_rn(sqrt_rn(iv), d);
        sums[0] = __fmaf_rn(v, d, sums[0]);
        sums[1] = __fmaf_rn(-v, -d, sums[1]);
        sums[2] = __fadd_rn(sums[2], log1pexp_naive(__fmul_rn(-zt, __fmul_rn(m, gy[i]))));
        sums[3] = __fadd_rn(sums[3], log1pexp_naive(__fmul_rn(zt, __fmul_rn(m, gx[i]))));
      }
      block_sum<4>(sums, red);
      const float n = (float)D;
      const float ratio = __fadd_rn(__fsub_rn(__fsub_rn(__fmul_rn(n, __fmul_rn(0.5f, sums[0])), sums[2]),
                                              __fmul_rn(n, __fmul_rn(0.5f, sums[1]))),
                                    sums[3]);
      la = __fadd_rn(__fsub_rn(logp_y, logp_x), ratio);
    }
    const float p_acc = clip_max1(expf(la));
    acc = uniform01(fold_in(rng(), 1u)) < p_acc;
    if (!loop) {
      if (A.info.proposal_position) big_store(A.info.proposal_position + ro, y, D);
      if (A.info.proposal_grad) big_store(A.info.proposal_grad + ro, gy, D);
    }
    if (tid == 0) {
      if (!loop) {
        if (A.info.proposal_logdensity) A.info.proposal_logdensity[c] = logp_y;
        if (A.info.acceptance_rate) A.info.acceptance_rate[c] = p_acc;
        if (A.info.is_accepted) A.info.is_accepted[c] = acc;
      } else if (A.acceptance_history) {
        A.acceptance_history[(size_t)t * P.C + c] = p_acc;
      }
    }
    if (acc) {  // each thread rewrites the elements it reads
      for (int i = tid; i < D; i += kBigThreads) {
        xs[i] = y[i];
        g_out[ro + i] = gy[i];
      }
      logp_x = logp_y;
    }
    __syncthreads();
    if (loop && BJX_KEEPS_HISTORY(A.loop, t)) big_store(BJX_HISTORY_ROW(A.loop, t, P.C, c, D), xs, D);
  }
  if (acc || loop) {
    big_store(q_out + ro, xs, D);
    if (tid == 0) logp_out[c] = logp_x;
  } else if (q_out != q_in) {  // an out-of-place rejection carries the old state over
    for (int i = tid; i < D / 4; i += kBigThreads) {
      __stcs(reinterpret_cast<float4*>(q_out + ro) + i, __ldcs(reinterpret_cast<const float4*>(q_in + ro) + i));
      __stcs(reinterpret_cast<float4*>(g_out + ro) + i, __ldcs(reinterpret_cast<const float4*>(g_in + ro) + i));
    }
    if (tid == 0) logp_out[c] = logp_x;
  }
}

// Elliptical slice transitions (the warp kernels' ess_transition_row, bjx_kernels.cuh) with a diagonal prior.  The
// proposal and its gradient scratch, which the target addresses freely, sit in shared memory; x and nu are read from
// global memory on every sub-iteration (nu from the [C, D] scratch A.nu), each thread using the elements t + 768 k that
// it writes itself: a third row of 18432 floats does not fit beside them.  One launch runs one transition
// (A.loop.step_keys == nullptr: keys and A.info as bjx_elliptical_slice_step's) or the A.loop.num_steps transitions of
// the native loop in place.
template <int TK>
__global__ void __launch_bounds__(kBigThreads) k_big_ess(BigParams P, const uint32_t* __restrict__ keys, const float* q_in,
                                                         const float* logl_in, float* q_out, float* logl_out, EssArgs A) {
  extern __shared__ __align__(16) float sm[];
  float *p = sm, *g = sm + P.D, *red = sm + 2 * (size_t)P.D;
  const int c = blockIdx.x, D = P.D, tid = threadIdx.x;
  const size_t ro = (size_t)c * D;
  const bool loop = A.loop.step_keys != nullptr;
  const int T = loop ? A.loop.num_steps : 1;
  const float* x = q_in + ro;  // the native loop: q_in == q_out, rewritten on acceptance
  float* nu = A.nu + ro;
  float logl_x = logl_in[c];
  for (int t = 0; t < T; ++t) {
    auto rng = [&]() {
      const uint32_t* kt = loop ? A.loop.step_keys + 2 * t : keys;
      return P.key_shared ? fold_in(Key{kt[0], kt[1]}, P.chain_offset + (uint32_t)c) : Key{kt[2 * c], kt[2 * c + 1]};
    };
    {
      const Key key_momentum = fold_in(rng(), 1u);
      for (int i = tid; i < D; i += kBigThreads)
        nu[i] = __fadd_rn(__ldg(A.mean + i), __fmul_rn(__ldg(A.scale + i), normal_at(key_momentum, (uint32_t)i)));
    }
    const float logy = __fadd_rn(logl_x, logf(uniform01(fold_in(rng(), 2u))));
    float theta = __fmul_rn(kEssTwoPi, uniform01(fold_in(rng(), 3u)));
    float theta_min = __fsub_rn(theta, kEssTwoPi), theta_max = theta;
    float sn, cs;
    auto propose = [&]() {
      ess_sincos(theta, sn, cs);
      for (int i = tid; i < D; i += kBigThreads) p[i] = ess_point(x[i], nu[i], __ldg(A.mean + i), cs, sn);
      __syncthreads();
      const float l = big_value_and_grad<TK>(P, p, g, red);
      __syncthreads();
      return l;
    };
    float logl_p = propose();
    int subiter = 1;
    while (logl_p <= logy && subiter < A.max_subiter) {
      const float f = uniform01(fold_in(fold_in(rng(), 0u), (uint32_t)subiter));
      theta = fmaxf(theta_min, __fadd_rn(__fmul_rn(f, __fsub_rn(theta_max, theta_min)), theta_min));
      logl_p = propose();
      if (theta < 0.f) theta_min = theta;
      if (theta > 0.f) theta_max = theta;
      ++subiter;
    }
    const bool exhausted = logl_p <= logy;
    if (!loop) {
      if (A.info.momentum)
        for (int i = tid; i < D; i += kBigThreads)
          A.info.momentum[ro + i] = exhausted ? nu[i] : ess_point(nu[i], x[i], __ldg(A.mean + i), cs, -sn);
      if (tid == 0) {
        if (A.info.theta) A.info.theta[c] = exhausted ? 0.f : theta;
        if (A.info.subiter) A.info.subiter[c] = subiter;
        if (A.info.exhausted) A.info.exhausted[c] = exhausted;
      }
    } else if (tid == 0 && A.subiter_history) {
      A.subiter_history[(size_t)t * P.C + c] = subiter;
    }
    if (!exhausted) {  // each thread rewrites the elements it reads
      for (int i = tid; i < D; i += kBigThreads) q_out[ro + i] = p[i];
      logl_x = logl_p;
      x = q_out + ro;
    } else if (q_out != q_in) {  // an out-of-place call carries the old state over
      for (int i = tid; i < D; i += kBigThreads) q_out[ro + i] = x[i];
    }
    if (loop && BJX_KEEPS_HISTORY(A.loop, t)) {
      float* hrow = BJX_HISTORY_ROW(A.loop, t, P.C, c, D);
      for (int i = tid; i < D; i += kBigThreads) hrow[i] = x[i];
    }
  }
  if (tid == 0) logl_out[c] = logl_x;
}


// Slice sampling transitions (the warp kernels' slice_transition_row and SliceMachine, bjx_kernels.cuh) with a [D]
// direction scale.  As in k_big_ess, the candidate x + t d and its gradient scratch sit in shared memory, x is re-read
// from its row on every evaluation and d lives in the [C, D] scratch A.dir, each thread using the elements t + 768 k
// that it writes itself.  One launch runs one transition (A.loop.step_keys == nullptr: keys and A.info as
// bjx_slice_step's) or the A.loop.num_steps transitions of the native loop in place.
template <int TK>
__global__ void __launch_bounds__(kBigThreads) k_big_slice(BigParams P, const uint32_t* __restrict__ keys, const float* q_in,
                                                           const float* logp_in, float* q_out, float* logp_out,
                                                           SliceArgs A) {
  extern __shared__ __align__(16) float sm[];
  float *p = sm, *g = sm + P.D, *red = sm + 2 * (size_t)P.D;
  const int c = blockIdx.x, D = P.D, tid = threadIdx.x;
  const size_t ro = (size_t)c * D;
  const bool loop = A.loop.step_keys != nullptr;
  const int T = loop ? A.loop.num_steps : 1;
  const float* x = q_in + ro;  // the native loop: q_in == q_out, rewritten on acceptance
  float* d = A.dir + ro;
  float logp_x = logp_in[c];
  unsigned long long evals = 0;
  for (int t = 0; t < T; ++t) {
    auto rng = [&]() {
      const uint32_t* kt = loop ? A.loop.step_keys + 2 * t : keys;
      return P.key_shared ? fold_in(Key{kt[0], kt[1]}, P.chain_offset + (uint32_t)c) : Key{kt[2 * c], kt[2 * c + 1]};
    };
    {  // d = n / |n|, n = 0 + scale z
      const Key prop_key = fold_in(rng(), 0u);
      float sq[1] = {0.f};
      for (int i = tid; i < D; i += kBigThreads) {
        const float v = __fadd_rn(0.f, __fmul_rn(__ldg(A.scale + i), normal_at(prop_key, (uint32_t)i)));
        d[i] = v;
        sq[0] = __fmaf_rn(v, v, sq[0]);
      }
      block_sum<1>(sq, red);
      const float nrm = sqrtf(sq[0]);
      for (int i = tid; i < D; i += kBigThreads) d[i] = __fdiv_rn(d[i], nrm);
    }
    const Key slice_key = fold_in(rng(), 1u);
    const float level = __fadd_rn(logp_x, logf(uniform01(fold_in(slice_key, 0u))));
    SliceMachine m;
    m.start(slice_key, P.eps_dev ? P.eps_dev[c] : P.eps, A);
    while (m.phase != SliceMachine::DONE) {
      for (int i = tid; i < D; i += kBigThreads) p[i] = __fadd_rn(x[i], __fmul_rn(m.x, d[i]));
      __syncthreads();
      const float lp = big_value_and_grad<TK>(P, p, g, red);
      __syncthreads();
      ++evals;
      m.feed(lp >= level, lp);
    }
    if (!loop) {
      if (tid == 0) {
        if (A.info.is_accepted) A.info.is_accepted[c] = m.found;
        if (A.info.num_expansions) A.info.num_expansions[c] = m.num_expansions;
        if (A.info.num_shrink) A.info.num_shrink[c] = m.n;
        if (A.info.bracket_left) A.info.bracket_left[c] = m.l;
        if (A.info.bracket_right) A.info.bracket_right[c] = m.r;
      }
    } else if (tid == 0) {
      if (A.expansions_history) A.expansions_history[(size_t)t * P.C + c] = m.num_expansions;
      if (A.shrink_history) A.shrink_history[(size_t)t * P.C + c] = m.n;
    }
    if (m.found) {  // each thread rewrites the elements it reads
      for (int i = tid; i < D; i += kBigThreads) q_out[ro + i] = __fadd_rn(x[i], __fmul_rn(m.t, d[i]));
      logp_x = m.lp_t;
      x = q_out + ro;
    } else if (q_out != q_in) {  // an out-of-place call carries the old state over
      for (int i = tid; i < D; i += kBigThreads) q_out[ro + i] = x[i];
    }
    if (loop && BJX_KEEPS_HISTORY(A.loop, t)) {
      float* hrow = BJX_HISTORY_ROW(A.loop, t, P.C, c, D);
      for (int i = tid; i < D; i += kBigThreads) hrow[i] = x[i];
    }
  }
  if (tid == 0) {
    logp_out[c] = logp_x;
    if (A.evaluations) atomicAdd(A.evaluations, evals);
  }
}

// Random-walk Metropolis transitions (the warp kernels' rw_transition_row, bjx_kernels.cuh) with a [D] sigma.  The
// proposal y and its gradient scratch, which the target addresses freely, sit in shared memory; x is re-read from its
// row, each thread using the elements t + 768 k that it also writes on acceptance.  One launch runs one transition
// (A.loop.step_keys == nullptr: keys and A.info as bjx_rw_step's) or the A.loop.num_steps transitions of the native loop
// in place.
template <int TK>
__global__ void __launch_bounds__(kBigThreads) k_big_rw(BigParams P, const uint32_t* __restrict__ keys, const float* q_in,
                                                        const float* logp_in, float* q_out, float* logp_out, RwArgs A) {
  extern __shared__ __align__(16) float sm[];
  float *y = sm, *g = sm + P.D, *red = sm + 2 * (size_t)P.D;
  const int c = blockIdx.x, D = P.D, tid = threadIdx.x;
  const size_t ro = (size_t)c * D;
  const bool loop = A.loop.step_keys != nullptr;
  const int T = loop ? A.loop.num_steps : 1;
  const bool independent = A.kind == RW_INDEPENDENT, correct = A.correct != 0;
  const float* x = q_in + ro;  // the native loop: q_in == q_out, rewritten on acceptance
  float logp_x = logp_in[c];
  for (int t = 0; t < T; ++t) {
    auto rng = [&]() {
      const uint32_t* kt = loop ? A.loop.step_keys + 2 * t : keys;
      return P.key_shared ? fold_in(Key{kt[0], kt[1]}, P.chain_offset + (uint32_t)c) : Key{kt[2 * c], kt[2 * c + 1]};
    };
    {
      const Key key_proposal = fold_in(rng(), 0u);
      for (int i = tid; i < D; i += kBigThreads) {
        const float lin = __fmul_rn(__ldg(A.sigma + i), normal_at(key_proposal, (uint32_t)i));
        y[i] = __fadd_rn(independent ? __ldg(A.mean + i) : x[i], lin);
      }
    }
    __syncthreads();
    const float logp_y = big_value_and_grad<TK>(P, y, g, red);
    __syncthreads();
    float sq[2] = {0.f, 0.f};  // sq_x, sq_y
    if (correct) {
      for (int i = tid; i < D; i += kBigThreads) {
        const float m = __ldg(A.mean + i), is = __ldg(A.inv_sigma + i);
        sq[0] = __fadd_rn(sq[0], rw_q_term(x[i], m, is));
        sq[1] = __fadd_rn(sq[1], rw_q_term(y[i], m, is));
      }
      block_sum<2>(sq, red);
    }
    const float p_acc = clip_max1(expf(rw_log_accept(logp_x, logp_y, correct, sq[0], sq[1])));
    const bool acc = uniform01(fold_in(rng(), 1u)) < p_acc;
    if (tid == 0) {
      if (!loop) {
        if (A.info.acceptance_rate) A.info.acceptance_rate[c] = p_acc;
        if (A.info.is_accepted) A.info.is_accepted[c] = acc;
      } else if (A.acceptance_history) {
        A.acceptance_history[(size_t)t * P.C + c] = p_acc;
      }
    }
    if (acc) {  // each thread rewrites the elements it reads
      for (int i = tid; i < D; i += kBigThreads) q_out[ro + i] = y[i];
      logp_x = logp_y;
      x = q_out + ro;
    } else if (q_out != q_in) {  // an out-of-place call carries the old state over
      for (int i = tid; i < D; i += kBigThreads) q_out[ro + i] = x[i];
    }
    if (loop && BJX_KEEPS_HISTORY(A.loop, t)) {
      float* hrow = BJX_HISTORY_ROW(A.loop, t, P.C, c, D);
      for (int i = tid; i < D; i += kBigThreads) hrow[i] = x[i];
    }
  }
  if (tid == 0) logp_out[c] = logp_x;
}

// ---- launch table shared by libbjx (built-in targets) and big-row plug-ins (TK = BJX_TARGET_USER) -------------------------
enum BigKernelId { BK_INIT = 0, BK_LEAPFROG = 1, BK_HMC = 2, BK_LANGEVIN = 3, BK_ESS = 4, BK_SLICE = 5, BK_RW = 6 };
struct BigLaunchArgs {
  BigParams P;
  const uint32_t* keys;
  const float *q_in, *logp_in, *g_in;
  float *q_out, *logp_out, *g_out;   // BK_INIT: logp_out, g_out; BK_LEAPFROG: q_out, logp_out, g_out in place (+ p_io)
  float* p_io;
  int n;                             // leapfrog steps | L
  InfoPtrs info;
  LangevinArgs langevin;             // BK_LANGEVIN
  EssArgs ess;                       // BK_ESS: q_in, logp_in (logL), q_out, logp_out
  SliceArgs slice;                   // BK_SLICE: q_in, logp_in, q_out, logp_out
  RwArgs rw;                         // BK_RW: q_in, logp_in, q_out, logp_out
  cudaStream_t stream;
};

// What a target plug-in must have been built against (bjx_plugin_abi, bjx_plugin_built_for_abi): the C ABI version and
// the layout of both launch-argument structs.
inline int plugin_abi() { return BJX_VERSION * 100000 + (int)sizeof(LaunchArgs) + 7 * (int)sizeof(BigLaunchArgs); }

// returns 0 or the cudaError_t of the attribute call / launch
template <int TK>
static int big_launch(int kernel_id, const BigLaunchArgs& a) {
  const int D = a.P.D, C = a.P.C;
  cudaStream_t st = a.stream;
  auto go = [&](auto kern, int rows, auto... args) -> int {
    const size_t smem = ((size_t)rows * D + 5 * kBigWarps) * sizeof(float);
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    kern<<<C, kBigThreads, smem, st>>>(args...);
    return (int)cudaGetLastError();
  };
  switch (kernel_id) {
    case BK_INIT:
      return go(k_big_init<TK>, 2, a.P, a.q_in, a.logp_out, a.g_out);
    case BK_LEAPFROG:
      if (D <= 14 * kBigThreads) return go(k_big_leapfrog<TK, 14>, 2, a.P, a.q_out, a.p_io, a.logp_out, a.g_out, a.n);
      return go(k_big_leapfrog<TK, 24>, 2, a.P, a.q_out, a.p_io, a.logp_out, a.g_out, a.n);
    case BK_HMC:
      return go(k_big_hmc<TK>, 3, a.P, a.keys, a.q_in, a.logp_in, a.g_in, a.q_out, a.logp_out, a.g_out, a.n, a.info);
    case BK_LANGEVIN:
      if (a.langevin.kind == LANGEVIN_MALA)
        return go(k_big_langevin<TK, LANGEVIN_MALA>, 3, a.P, a.keys, a.q_in, a.logp_in, a.g_in, a.q_out, a.logp_out,
                  a.g_out, a.langevin);
      return go(k_big_langevin<TK, LANGEVIN_BARKER>, 3, a.P, a.keys, a.q_in, a.logp_in, a.g_in, a.q_out, a.logp_out,
                a.g_out, a.langevin);
    case BK_ESS:
      return go(k_big_ess<TK>, 2, a.P, a.keys, a.q_in, a.logp_in, a.q_out, a.logp_out, a.ess);
    case BK_SLICE:
      return go(k_big_slice<TK>, 2, a.P, a.keys, a.q_in, a.logp_in, a.q_out, a.logp_out, a.slice);
    case BK_RW:
      return go(k_big_rw<TK>, 2, a.P, a.keys, a.q_in, a.logp_in, a.q_out, a.logp_out, a.rw);
    default:
      return (int)cudaErrorInvalidValue;
  }
}
}  // namespace bjx
