// Warp-owns-a-chain row primitives for the HMC/NUTS kernels.
//
// Layout: state arrays are float32 [C, D] row-major.  One warp owns one chain row; lane l holds
// NS "slots" of the row in registers.  VEC layout (D % 4 == 0): slot s = 4*j + v is element
// (j*32 + l)*4 + v, so each j is one coalesced 512-byte LDG.128/STG.128 per warp.  Scalar layout
// (any D <= 32*NS): slot s is element s*32 + l.  Slots past D are held as 0 so that per-chain
// reductions (log-density, kinetic energy, U-turn dot products) need no masks and finish with
// __shfl_xor_sync inside the owning warp -- no shared memory, no cross-CTA traffic.
//
// Rounding: the integrator updates `x + (eps*coef)*grad` (blackjax/mcmc/integrators.py:200,236) are
// compiled with FMA contraction (nvcc default -fmad=true), i.e. one fused multiply-add per update.
// That is also what the reference's own CPU backend does: XLA:CPU builds its LLVM target with
// AllowFPOpFusion = Fast ("always allow FMA fusion"), so on an FMA-capable host the same expression
// lowers to vfmadd.  The oracle emulates the contraction (oracle/hmc.py FMA_CONTRACT) so purely
// elementwise targets stay bit-comparable; everything is within the 1e-5 tolerance either way.
// PRNG transforms use explicit round-to-nearest intrinsics and are unaffected.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "bjx_prng.cuh"

namespace bjx {

enum { TK_DIAG = 0, TK_FUNNEL = 1, TK_DENSE = 2, TK_BANANA = 3, TK_USER = 4 };

// kernels whose warps need a D-float shared-memory slice (small dense matvec staging; scratch of user-defined targets)
template <int TK, bool DM>
__host__ __device__ constexpr bool needs_row_smem() { return DM || TK == TK_DENSE || TK == TK_USER; }

struct Params {
  int C, D;
  // target
  const float* inv_var;
  const float* mean;
  const float* prec;
  float logp_offset;
  const float* user;       // TK_USER: the user's parameter block (n_user floats: data, hyper-parameters)
  int n_user;
  // metric
  const float* imm;        // diag: [D] or [C,D]; dense: [D,D]
  long long imm_stride;    // 0 (shared), D (one row per group of imm_group chains) or D*D (one dense matrix per chain)
  int imm_group;           // chains sharing a metric row (1: per chain; MEADS folds: chains per fold)
  const float* msqrt;      // mass_matrix_sqrt, same layout as imm
  // low-rank metric (metrics.py:349-467): M^-1 = diag(sigma) (I + U (Lambda - I) U^T) diag(sigma); lr_k == 0: not in use
  int lr_k;
  const float* lr_U;        // [D, k] row-major, orthonormal columns
  const float* lr_sigma;    // [D]
  const float* lr_inv_sigma;
  const float* lr_lam_m1;   // [k] lambda - 1
  const float* lr_isl_m1;   // [k] 1/sqrt(lambda) - 1
  // step size
  float eps;
  const float* eps_dev;    // [C] or nullptr
  float div_thr;
  // PRNG key source: per-chain keys [C,2] (key_shared == 0) or ONE step key [2] from which chain c derives
  // split(step_key, n_global)[chain_offset + c] = fold_in(step_key, chain_offset + c) in-kernel (key_shared == 1):
  // the reference's step-major schedule (howto_sample_multiple_chains.md:116-129) without a separate split launch,
  // and invariant to how the chains are sharded over GPUs.
  int key_shared;
  uint32_t chain_offset;
  // per-chain number of integration steps (dynamic HMC, mcmc/dynamic_hmc.py:109-120) or nullptr (the launch's scalar L)
  const int* steps_dev;
  // palindromic two-stage integrator coefficients (integrators.py:62-152); velocity Verlet = {0.5, 1, 0.5}
  int ncoef;
  float coef[11];
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- paired elementwise FP32 ops: explicit IEEE round-to-nearest, never contracted ----
// Every elementwise update below goes through these helpers on pairs of adjacent slots (odd slot counts use
// plain scalar ops), with the dot products keeping two interleaved accumulators.  The _rn intrinsics stop the
// compiler from fusing a product into a later add, so each result is the one rounded operation written here.
__device__ __forceinline__ void fma2(float& d0, float& d1, float a0, float a1, float b0, float b1, float c0, float c1) {
  d0 = __fmaf_rn(a0, b0, c0);
  d1 = __fmaf_rn(a1, b1, c1);
}
__device__ __forceinline__ void mul2(float& d0, float& d1, float a0, float a1, float b0, float b1) {
  d0 = __fmul_rn(a0, b0);
  d1 = __fmul_rn(a1, b1);
}
__device__ __forceinline__ void add2(float& d0, float& d1, float a0, float a1, float b0, float b1) {
  d0 = __fadd_rn(a0, b0);
  d1 = __fadd_rn(a1, b1);
}

// ---- user-defined targets (TK_USER; include/bjx_user_target.h) -----------------------------------------------------
// BlackJAX differentiates any `logdensity_fn` with jax.value_and_grad (mcmc/hmc.py:91, integrators.py:189).  Without a
// tracing compiler the plug-in point is the fused value_and_grad itself: the user writes ONE small device struct against the
// row layout above; bjx_plugin.cu instantiates every transition kernel of the path around it (nvcc, one small .so per
// target) and libbjx dispatches to it like to a built-in target.
struct UserCtx {
  const float* theta;  // parameter block [n_theta] (device memory, read-only)
  int n_theta;
  int D;               // row length; slots with Row::idx(s, lane) >= D hold 0 on entry and must be left 0 in g
  int lane;
  float* row_smem;     // this warp's scratch of D floats in shared memory (see row_stage)
};
}  // namespace bjx
namespace bjx_user {
// The user's model, defined by the plug-in's source (never by libbjx itself):
//   template <class R> struct Model {
//     /* per-kernel state in registers, e.g. float w[R::NS]; */
//     __device__ __forceinline__ void init(const bjx::UserCtx& u);            // once per kernel launch and chain row
//     template <bool WANT_LOGP>
//     __device__ __forceinline__ void value_and_grad(const bjx::UserCtx& u, const float (&q)[R::NS], float (&g)[R::NS],
//                                                    float& logp) const;
//   };
// value_and_grad: q[s] / g[s] are the slots of this lane (element index R::idx(s, lane)); logp must come back identical on
// all lanes when WANT_LOGP (otherwise it is dead and the reduction may be skipped).
template <class R>
struct Model;
}  // namespace bjx_user
namespace bjx {

template <int NS>
struct Vec {
  // x = fma(a, y, x)
  __device__ static __forceinline__ void axpy(float (&x)[NS], float a, const float (&y)[NS]) {
    if constexpr (NS % 2 == 0) {
#pragma unroll
      for (int s = 0; s < NS; s += 2) fma2(x[s], x[s + 1], a, a, y[s], y[s + 1], x[s], x[s + 1]);
    } else {
#pragma unroll
      for (int s = 0; s < NS; ++s) x[s] = fmaf(a, y[s], x[s]);
    }
  }
  // d = a * b
  __device__ static __forceinline__ void mul(float (&d)[NS], const float (&a)[NS], const float (&b)[NS]) {
    if constexpr (NS % 2 == 0) {
#pragma unroll
      for (int s = 0; s < NS; s += 2) mul2(d[s], d[s + 1], a[s], a[s + 1], b[s], b[s + 1]);
    } else {
#pragma unroll
      for (int s = 0; s < NS; ++s) d[s] = a[s] * b[s];
    }
  }
  // d = a * b (scalar a)
  __device__ static __forceinline__ void scale(float (&d)[NS], float a, const float (&b)[NS]) {
    if constexpr (NS % 2 == 0) {
#pragma unroll
      for (int s = 0; s < NS; s += 2) mul2(d[s], d[s + 1], a, a, b[s], b[s + 1]);
    } else {
#pragma unroll
      for (int s = 0; s < NS; ++s) d[s] = a * b[s];
    }
  }
  // d = a + b
  __device__ static __forceinline__ void add(float (&d)[NS], const float (&a)[NS], const float (&b)[NS]) {
    if constexpr (NS % 2 == 0) {
#pragma unroll
      for (int s = 0; s < NS; s += 2) add2(d[s], d[s + 1], a[s], a[s + 1], b[s], b[s + 1]);
    } else {
#pragma unroll
      for (int s = 0; s < NS; ++s) d[s] = a[s] + b[s];
    }
  }
  // per-lane partial of sum_s a[s]*b[s] (two interleaved accumulators when packed)
  __device__ static __forceinline__ float dot_partial(const float (&a)[NS], const float (&b)[NS]) {
    if constexpr (NS % 2 == 0) {
      float e = 0.f, o = 0.f;
#pragma unroll
      for (int s = 0; s < NS; s += 2) fma2(e, o, a[s], a[s + 1], b[s], b[s + 1], e, o);
      return e + o;
    } else {
      float acc = 0.f;
#pragma unroll
      for (int s = 0; s < NS; ++s) acc = fmaf(a[s], b[s], acc);
      return acc;
    }
  }
};

template <int NS_, bool VEC_>
struct Row {
  static constexpr int NS = NS_;
  static constexpr bool VEC = VEC_;
  static_assert(!VEC_ || (NS_ % 4 == 0), "vector layout needs NS % 4 == 0");

  __device__ static __forceinline__ int idx(int s, int lane) {
    return VEC ? (((s >> 2) * 32 + lane) * 4 + (s & 3)) : (s * 32 + lane);
  }

  // streaming (evict-first) loads/stores for the [C,D] state arrays
  __device__ static __forceinline__ void load(float (&x)[NS], const float* __restrict__ row, int D, int lane) {
    if constexpr (VEC) {
#pragma unroll
      for (int j = 0; j < NS / 4; ++j) {
        const int e = (j * 32 + lane) * 4;
        float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
        if (e < D) t = __ldcs(reinterpret_cast<const float4*>(row + e));
        x[4 * j + 0] = t.x; x[4 * j + 1] = t.y; x[4 * j + 2] = t.z; x[4 * j + 3] = t.w;
      }
    } else {
#pragma unroll
      for (int s = 0; s < NS; ++s) {
        const int e = s * 32 + lane;
        x[s] = (e < D) ? __ldcs(row + e) : 0.f;
      }
    }
  }
  // cached loads for small shared vectors (inverse mass, target scales)
  __device__ static __forceinline__ void load_const(float (&x)[NS], const float* __restrict__ row, int D, int lane) {
    if constexpr (VEC) {
#pragma unroll
      for (int j = 0; j < NS / 4; ++j) {
        const int e = (j * 32 + lane) * 4;
        float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
        if (e < D) t = __ldg(reinterpret_cast<const float4*>(row + e));
        x[4 * j + 0] = t.x; x[4 * j + 1] = t.y; x[4 * j + 2] = t.z; x[4 * j + 3] = t.w;
      }
    } else {
#pragma unroll
      for (int s = 0; s < NS; ++s) {
        const int e = s * 32 + lane;
        x[s] = (e < D) ? __ldg(row + e) : 0.f;
      }
    }
  }
  __device__ static __forceinline__ void store(const float (&x)[NS], float* __restrict__ row, int D, int lane) {
    if constexpr (VEC) {
#pragma unroll
      for (int j = 0; j < NS / 4; ++j) {
        const int e = (j * 32 + lane) * 4;
        if (e < D) __stcs(reinterpret_cast<float4*>(row + e), make_float4(x[4 * j], x[4 * j + 1], x[4 * j + 2], x[4 * j + 3]));
      }
    } else {
#pragma unroll
      for (int s = 0; s < NS; ++s) {
        const int e = s * 32 + lane;
        if (e < D) __stcs(row + e, x[s]);
      }
    }
  }
  // plain (generic-address) store: the destination may be shared memory (NUTS checkpoints)
  __device__ static __forceinline__ void store_generic(const float (&x)[NS], float* row, int D, int lane) {
    if constexpr (VEC) {
#pragma unroll
      for (int j = 0; j < NS / 4; ++j) {
        const int e = (j * 32 + lane) * 4;
        if (e < D) *reinterpret_cast<float4*>(row + e) = make_float4(x[4 * j], x[4 * j + 1], x[4 * j + 2], x[4 * j + 3]);
      }
    } else {
#pragma unroll
      for (int s = 0; s < NS; ++s) {
        const int e = s * 32 + lane;
        if (e < D) row[e] = x[s];
      }
    }
  }
  __device__ static __forceinline__ void load_generic(float (&x)[NS], const float* row, int D, int lane) {
    if constexpr (VEC) {
#pragma unroll
      for (int j = 0; j < NS / 4; ++j) {
        const int e = (j * 32 + lane) * 4;
        float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
        if (e < D) t = *reinterpret_cast<const float4*>(row + e);
        x[4 * j + 0] = t.x; x[4 * j + 1] = t.y; x[4 * j + 2] = t.z; x[4 * j + 3] = t.w;
      }
    } else {
#pragma unroll
      for (int s = 0; s < NS; ++s) {
        const int e = s * 32 + lane;
        x[s] = (e < D) ? row[e] : 0.f;
      }
    }
  }
  __device__ static __forceinline__ float dot(const float (&a)[NS], const float (&b)[NS]) {
    return warp_sum(Vec<NS>::dot_partial(a, b));
  }
};

// y = M x for a small dense [D,D] matrix: the warp stages x in its shared-memory slice and each
// lane forms the rows it owns.  Used for dense metrics/targets with D <= 128 (KAT-sized problems);
// large dense problems go through the batched GEMM path instead.
template <class R>
__device__ __forceinline__ void matvec_small(const float* __restrict__ M, const float (&x)[R::NS], float (&y)[R::NS],
                                             float* sm, int D, int lane) {
#pragma unroll
  for (int s = 0; s < R::NS; ++s) {
    const int e = R::idx(s, lane);
    if (e < D) sm[e] = x[s];
  }
  __syncwarp();
#pragma unroll
  for (int s = 0; s < R::NS; ++s) {
    const int e = R::idx(s, lane);
    float acc = 0.f;
    if (e < D) {
      const float* mr = M + (size_t)e * D;
      for (int j = 0; j < D; ++j) acc = fmaf(__ldg(mr + j), sm[j], acc);
    }
    y[s] = acc;
  }
  __syncwarp();
}

// Helpers for user-defined targets: random access to the row.
// row_stage: copy the row into the warp's shared-memory scratch (element e at u.row_smem[e]); every lane can then read
// any element.  row_at<E>: broadcast element E (compile-time index) straight from the owner's register.
template <class R>
__device__ __forceinline__ void row_stage(const UserCtx& u, const float (&x)[R::NS]) {
  __syncwarp();
#pragma unroll
  for (int s = 0; s < R::NS; ++s) {
    const int e = R::idx(s, u.lane);
    if (e < u.D) u.row_smem[e] = x[s];
  }
  __syncwarp();
}
template <class R, int E>
__device__ __forceinline__ float row_at(const float (&x)[R::NS]) {
  constexpr int slot = R::VEC ? ((E >> 7) * 4 + (E & 3)) : (E >> 5);
  constexpr int owner = R::VEC ? ((E & 127) >> 2) : (E & 31);
  static_assert(slot < R::NS, "element index beyond the row");
  return __shfl_sync(0xffffffffu, x[slot], owner);
}

// y = x + U ((s - 1) (U^T x))   (_low_rank_matvec, metrics.py:131-177) for a row held by one warp: every lane forms its
// part of the k <= 16 projections, k interleaved shuffle reductions, then the expansion -- O(D k / 32) per lane, U read
// through the read-only path (D k floats: L1/L2 resident).
constexpr int kMaxLowRank = 16;
template <class R>
__device__ __forceinline__ void lowrank_apply(const float* __restrict__ U, const float* __restrict__ sm1, int k,
                                              const float (&x)[R::NS], float (&y)[R::NS], int D, int lane) {
#pragma unroll
  for (int s = 0; s < R::NS; ++s) y[s] = x[s];
  // four projections at a time: their shuffle reductions interleave, and the code stays small (the operator is inlined
  // at every velocity / kinetic-energy / momentum-draw site of every kernel)
  for (int j0 = 0; j0 < k; j0 += 4) {
    float t[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int s = 0; s < R::NS; ++s) {
      const int e = R::idx(s, lane);
      if (e < D) {
        const float* ur = U + (size_t)e * k + j0;
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if (j0 + u < k) t[u] = fmaf(__ldg(ur + u), x[s], t[u]);
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) t[u] = (j0 + u < k) ? warp_sum(t[u]) * __ldg(sm1 + j0 + u) : 0.f;
#pragma unroll
    for (int s = 0; s < R::NS; ++s) {
      const int e = R::idx(s, lane);
      if (e < D) {
        const float* ur = U + (size_t)e * k + j0;
        float a = 0.f;
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if (j0 + u < k) a = fmaf(__ldg(ur + u), t[u], a);
        y[s] += a;
      }
    }
  }
}

struct NoUserModel {};
template <class R, int TK>
struct UserModelOf { using type = NoUserModel; };
template <class R>
struct UserModelOf<R, TK_USER> { using type = bjx_user::Model<R>; };

// Per-warp constant context: target scales and inverse mass held in registers for the whole kernel.
// MSM: the diagonal inverse mass and the diagonal target's scales live in the warp's shared-memory rows msm and tsm (set
// before init) instead of registers, for kernels that need those registers; the products are the same.
template <class R, int TK, bool DM, bool MSM = false>
struct Ctx {
  typename UserModelOf<R, TK>::type um;   // TK_USER: the user's model (its per-kernel state lives here)
  float tw[(TK == TK_DIAG && !MSM) ? R::NS : 1];  // target -1/s^2 (negated once: grad = q * tw, exactly -(q/s^2))
  float mw[(DM || MSM) ? 1 : R::NS];      // diagonal inverse mass
  float *msm, *tsm;                       // MSM: the diagonal inverse mass and target rows in shared memory
  float* sm;                              // shared-memory slice (small dense paths)
  size_t moff;                            // small dense metric: offset of this chain's matrix (0 when shared)
  int lane;

  __device__ __forceinline__ void init(const Params& P, int chain, int lane_, float* sm_) {
    lane = lane_;
    sm = sm_;
    if constexpr (TK == TK_DIAG && MSM) {
      float t[R::NS];
      R::load_const(t, P.inv_var, P.D, lane);
#pragma unroll
      for (int s = 0; s < R::NS; ++s) t[s] = -t[s];
      __syncwarp();
      R::store_generic(t, tsm, P.D, lane);
      __syncwarp();
    } else if constexpr (TK == TK_DIAG) {
      R::load_const(tw, P.inv_var, P.D, lane);
#pragma unroll
      for (int s = 0; s < R::NS; ++s) tw[s] = -tw[s];
    }
    if constexpr (TK == TK_USER) um.init(UserCtx{P.user, P.n_user, P.D, lane, sm});
    moff = 0;
    if constexpr (!DM && MSM) {
      float t[R::NS];
      R::load_const(t, P.imm + (size_t)(chain / P.imm_group) * P.imm_stride, P.D, lane);
      __syncwarp();
      R::store_generic(t, msm, P.D, lane);
      __syncwarp();
    } else if constexpr (!DM) R::load_const(mw, P.imm + (size_t)(chain / P.imm_group) * P.imm_stride, P.D, lane);
    else moff = (size_t)(chain / P.imm_group) * P.imm_stride;  // D*D per chain for per-chain dense metrics
  }

  // linear_map(M^-1, p)   blackjax/util.py:57-61
  __device__ __forceinline__ void velocity(const Params& P, const float (&p)[R::NS], float (&v)[R::NS]) {
    if constexpr (DM) {
      if (P.lr_k > 0) {  // sigma * lowrank(sigma * p, lambda)   metrics.py:430-432
        float sg[R::NS], qv[R::NS];
        R::load_const(sg, P.lr_sigma, P.D, lane);
        Vec<R::NS>::mul(qv, sg, p);
        lowrank_apply<R>(P.lr_U, P.lr_lam_m1, P.lr_k, qv, v, P.D, lane);
        Vec<R::NS>::mul(v, sg, v);
      } else if constexpr (R::NS <= 4) {  // small dense metrics exist for dim <= 128 only
        matvec_small<R>(P.imm + moff, p, v, sm, P.D, lane);
      }
    } else if constexpr (MSM) {
      R::load_generic(v, msm, P.D, lane);  // each lane reads back the slots it wrote
      Vec<R::NS>::mul(v, v, p);
    } else {
      Vec<R::NS>::mul(v, mw, p);
    }
  }

  // kinetic_energy  blackjax/mcmc/metrics.py:263-270: 0.5 * dot(M^-1 p, p)
  __device__ __forceinline__ float kinetic(const Params& P, const float (&p)[R::NS]) {
    float v[R::NS];
    if constexpr (DM) {
      if (P.lr_k > 0) {  // 0.5 * dot(q, lowrank(q, lambda)), q = sigma * p   metrics.py:401-408
        float sg[R::NS], qv[R::NS];
        R::load_const(sg, P.lr_sigma, P.D, lane);
        Vec<R::NS>::mul(qv, sg, p);
        lowrank_apply<R>(P.lr_U, P.lr_lam_m1, P.lr_k, qv, v, P.D, lane);
        return 0.5f * R::dot(qv, v);
      }
    }
    velocity(P, p, v);
    return 0.5f * R::dot(v, p);
  }

  // value_and_grad of the target at q.  WANT_LOGP=false skips the log-density reduction where only the
  // gradient is consumed (interior steps of a fixed-length trajectory: the value is dead there).
  template <bool WANT_LOGP = true>
  __device__ __forceinline__ void value_and_grad(const Params& P, const float (&q)[R::NS], float (&g)[R::NS], float& logp) {
    if constexpr (TK == TK_DIAG) {
      // g = (q - mean) * (-1/s^2);  logp = 0.5 * sum (q - mean) * g   (negation is exact, so this equals
      // -0.5 * sum d * (d / s^2) bit for bit)
      float acc;
      if (P.mean != nullptr) {
        float d[R::NS];
        R::load_const(d, P.mean, P.D, lane);
#pragma unroll
        for (int s = 0; s < R::NS; ++s) d[s] = -d[s];
        Vec<R::NS>::add(d, q, d);
        if constexpr (MSM) {
          R::load_generic(g, tsm, P.D, lane);
          Vec<R::NS>::mul(g, d, g);
        } else {
          Vec<R::NS>::mul(g, d, tw);
        }
        acc = WANT_LOGP ? Vec<R::NS>::dot_partial(d, g) : 0.f;
      } else if constexpr (MSM) {
        R::load_generic(g, tsm, P.D, lane);
        Vec<R::NS>::mul(g, q, g);
        acc = WANT_LOGP ? Vec<R::NS>::dot_partial(q, g) : 0.f;
      } else {
        Vec<R::NS>::mul(g, q, tw);
        acc = WANT_LOGP ? Vec<R::NS>::dot_partial(q, g) : 0.f;
      }
      if (WANT_LOGP) logp = 0.5f * warp_sum(acc) + P.logp_offset;
    } else if constexpr (TK == TK_FUNNEL) {
      const float y = __shfl_sync(0xffffffffu, q[0], 0);
      const float q0 = q[0];
      {  // sum of v^2 over the funnel coordinates (the neck slot contributes an exact 0)
        float qq[R::NS];
#pragma unroll
        for (int s = 0; s < R::NS; ++s) qq[s] = q[s];
        if (lane == 0) qq[0] = 0.f;
        const float ss = warp_sum(Vec<R::NS>::dot_partial(qq, qq));
        const float ey = expf(-y);
        const float n = (float)(P.D - 1);
        const float t = y / 3.0f;
        logp = -0.5f * (t * t) + (-0.5f * ey * ss - 0.5f * n * y) + P.logp_offset;
        Vec<R::NS>::scale(g, -ey, q);
        if (lane == 0) g[0] = -q0 / 9.0f + 0.5f * ey * ss - 0.5f * n;
      }
    } else if constexpr (TK == TK_DENSE) {
      matvec_small<R>(P.prec, q, g, sm, P.D, lane);
      logp = -0.5f * R::dot(q, g) + P.logp_offset;
#pragma unroll
      for (int s = 0; s < R::NS; ++s) g[s] = -g[s];
    } else if constexpr (TK == TK_USER) {
      const UserCtx u{P.user, P.n_user, P.D, lane, sm};
      float lp = 0.f;
      um.template value_and_grad<WANT_LOGP>(u, q, g, lp);
      if (WANT_LOGP) logp = lp + P.logp_offset;
      __syncwarp();  // the scratch slice is shared with the small dense metric's matvec
    } else {  // TK_BANANA, D == 2, scalar layout: x0 at lane 0, x1 at lane 1
      const float x0 = __shfl_sync(0xffffffffu, q[0], 0);
      const float x1 = __shfl_sync(0xffffffffu, q[0], 1);
      const float r = x1 - x0 * x0;
      const float a = 1.0f - x0;
      logp = -(a * a) - 1.5f * r * r + P.logp_offset;
#pragma unroll
      for (int s = 0; s < R::NS; ++s) g[s] = 0.f;
      if (lane == 0) g[0] = 2.0f * a + 6.0f * r * x0;
      if (lane == 1) g[0] = -3.0f * r;
    }
  }

  // one velocity-Verlet step, coefficients [0.5, 1.0, 0.5]
  // (blackjax/mcmc/integrators.py:104-150,199-203,235-245,321-322)
  template <bool WANT_LOGP = true>
  __device__ __forceinline__ void leapfrog(const Params& P, float (&q)[R::NS], float (&p)[R::NS], float (&g)[R::NS],
                                           float& logp, float eps) {
    const float eh = eps * 0.5f;
    const float e1 = eps * 1.0f;
    Vec<R::NS>::axpy(p, eh, g);
    {
      float v[R::NS];
      velocity(P, p, v);
      Vec<R::NS>::axpy(q, e1, v);
    }
    value_and_grad<WANT_LOGP>(P, q, g, logp);
    Vec<R::NS>::axpy(p, eh, g);
  }

  // generalized_two_stage_integrator (integrators.py:104-150) for an arbitrary palindromic coefficient table
  // (mclachlan / yoshida / omelyan, integrators.py:335-369): even entries kick the momentum, odd entries drift
  // the position and re-evaluate the gradient; the last kick skips the kinetic gradient.
  template <bool WANT_LOGP = true>
  __device__ __forceinline__ void integrate_general(const Params& P, float (&q)[R::NS], float (&p)[R::NS],
                                                    float (&g)[R::NS], float& logp, float eps) {
    for (int i = 0; i + 1 < P.ncoef; ++i) {
      const float a = eps * P.coef[i];
      if ((i & 1) == 0) {
        Vec<R::NS>::axpy(p, a, g);
      } else {
        float v[R::NS];
        velocity(P, p, v);  // kinetic_grad of the momentum just updated (integrators.py:242)
        Vec<R::NS>::axpy(q, a, v);
        if (WANT_LOGP || i + 2 < P.ncoef) value_and_grad<true>(P, q, g, logp);
        else value_and_grad<false>(P, q, g, logp);
      }
    }
    Vec<R::NS>::axpy(p, eps * P.coef[P.ncoef - 1], g);
  }

  // one integrator step: velocity Verlet fast path or the general coefficient table
  template <bool GEN, bool WANT_LOGP = true>
  __device__ __forceinline__ void step(const Params& P, float (&q)[R::NS], float (&p)[R::NS], float (&g)[R::NS],
                                       float& logp, float eps) {
    if constexpr (GEN) integrate_general<WANT_LOGP>(P, q, p, g, logp, eps);
    else leapfrog<WANT_LOGP>(P, q, p, g, logp, eps);
  }

  // metric.sample_momentum  metrics.py:260-261 -> util.py:89-91: p = mass_matrix_sqrt (.) normal(key,(D,))
  __device__ __forceinline__ void sample_momentum(const Params& P, int chain, Key key, float (&p)[R::NS]) {
    float z[R::NS];
#pragma unroll
    for (int s = 0; s < R::NS; ++s) {
      const int e = R::idx(s, lane);
      z[s] = (e < P.D) ? normal_at(key, (uint32_t)e) : 0.f;
    }
    if constexpr (DM) {
      if (P.lr_k > 0) {  // (1/sigma) * lowrank(eps, 1/sqrt(lambda))   metrics.py:389-399
        float is[R::NS];
        lowrank_apply<R>(P.lr_U, P.lr_isl_m1, P.lr_k, z, p, P.D, lane);
        R::load_const(is, P.lr_inv_sigma, P.D, lane);
        Vec<R::NS>::mul(p, is, p);
      } else if constexpr (R::NS <= 4) {
        matvec_small<R>(P.msqrt + moff, z, p, sm, P.D, lane);
      }
    } else {
      float ms[R::NS];
      R::load_const(ms, P.msqrt + (size_t)(chain / P.imm_group) * P.imm_stride, P.D, lane);
#pragma unroll
      for (int s = 0; s < R::NS; ++s) p[s] = ms[s] * z[s];
    }
  }

  // gaussian_euclidean.is_turning  metrics.py:272-304 (<=, OR)
  __device__ __forceinline__ bool is_turning(const Params& P, const float (&pl)[R::NS], const float (&pr)[R::NS],
                                             const float (&psum)[R::NS]) {
    float rho[R::NS], v[R::NS];
#pragma unroll
    for (int s = 0; s < R::NS; ++s) rho[s] = psum[s] - (pr[s] + pl[s]) / 2.0f;
    velocity(P, pl, v);
    const float dl = R::dot(v, rho);
    velocity(P, pr, v);
    const float dr = R::dot(v, rho);
    return (dl <= 0.f) || (dr <= 0.f);
  }
};

__device__ __forceinline__ Key chain_key(const Params& P, const uint32_t* __restrict__ keys, int chain) {
  if (P.key_shared) return fold_in(Key{keys[0], keys[1]}, P.chain_offset + (uint32_t)chain);
  return Key{keys[2 * chain], keys[2 * chain + 1]};
}

__device__ __forceinline__ float safe_energy_diff(float e0, float e1) {  // proposal.py:45-48
  const float d = e0 - e1;
  return isnan(d) ? -__int_as_float(0x7f800000) : d;
}

__device__ __forceinline__ float logaddexp_f(float a, float b) {  // jnp.logaddexp
  const float amax = fmaxf(a, b);
  const float delta = a - b;
  if (isnan(delta)) return a + b;
  return amax + log1pf(expf(-fabsf(delta)));
}

__device__ __forceinline__ float expit_f(float x) { return 1.0f / (1.0f + expf(-x)); }  // jax.scipy.special.expit

}  // namespace bjx
