// Template dispatch: (target kind, size class, dense-small metric) -> kernel instantiation.
// Each target kind is instantiated in its own translation unit (bjx_inst_*.cu) so the build
// parallelises; bjx_api.cu only sees the declaration of Launcher<TK>::launch.
#pragma once
#include <algorithm>

#include "bjx_internal.h"
#include "bjx_kernels.cuh"

namespace bjx {

enum SizeClass { SC_V1 = 0, SC_V2, SC_V4, SC_V8, SC_S1, SC_S4, SC_BIG, SC_NONE };  // SC_BIG: CTA-per-chain (bjx_big.cu)
enum KernelId { K_INIT = 0, K_MOMENTUM, K_LEAPFROG, K_ENERGY, K_TURNING, K_HMC, K_NUTS_INIT, K_NUTS_DOUBLING, K_MHMC, K_GHMC, K_NUTS_CHAINS,
               K_MCLMC, K_AMCLMC, K_MCLMC_TUNE, K_AMCLMC_TUNE, K_LAPS_BURN_IN, K_GIST, K_GIST_CHAINS, K_LANGEVIN,
               K_LANGEVIN_CHAINS, K_ESS, K_ESS_CHAINS, K_SLICE, K_SLICE_CHAINS, K_RW, K_RW_CHAINS };

struct LaunchArgs {
  Params P;
  NutsWs ws;
  InfoPtrs info;
  GhmcArgs ghmc;
  NutsSampleArgs sample;
  MclmcArgs mclmc;
  AmclmcArgs amclmc;
  MclmcTuneArgs mclmc_tune;
  AmclmcTuneArgs amclmc_tune;
  LapsArgs laps;
  GistArgs gist;
  LangevinArgs langevin;
  EssArgs ess;         // K_ESS / K_ESS_CHAINS: q_in, logp_in (logL), q_out, logp_out
  SliceArgs slice;     // K_SLICE / K_SLICE_CHAINS: q_in, logp_in, q_out, logp_out
  RwArgs rw;           // K_RW / K_RW_CHAINS: q_in, logp_in, q_out, logp_out
  const uint32_t* keys;
  const float *q_in, *logp_in, *g_in;
  float *q_out, *logp_out, *g_out;
  float* p_io;
  int n;  // n_steps | L | max_doublings
  int depth;            // first doubling of this launch
  int depth_end;        // one past the last doubling of this launch
  int ckpt_smem;        // checkpoints in shared memory
  const int* list_in;   // compacted chain indices (nullptr = identity)
  int n_in;             // number of warps to launch (0 = all chains)
  const int* n_in_dev;  // device-side row count (then n_in is only the grid's upper bound)
  int* list_out;
  int* counter;
  const float* mom_override;
  const uint32_t* keyint_override;
  float* mom_out;
  const float *pl, *pr, *ps;
  uint8_t* out_u8;
  float* e_out;
  bool general_integrator;  // coefficient table other than velocity Verlet
  cudaStream_t stream;
};

inline SizeClass size_class_for(int D) {
  if (D <= 0) return SC_NONE;
  if (D % 4 == 0 && D <= 1024) return D <= 128 ? SC_V1 : D <= 256 ? SC_V2 : D <= 512 ? SC_V4 : SC_V8;
  if (D <= 32) return SC_S1;
  if (D <= 128) return SC_S4;
  if (D % 4 == 0 && D <= 18432) return SC_BIG;
  return SC_NONE;
}
inline bool size_class_is_small(int sc) { return sc == SC_V1 || sc == SC_S1 || sc == SC_S4; }
inline bool size_class_is_vec(int sc) { return sc <= SC_V8 || sc == SC_BIG; }

template <int TK>
struct Launcher {
  // returns 0, or -2 when the combination is not built
  static int launch(int kernel_id, int sc, bool dm, const LaunchArgs& a);
};

#ifdef BJX_INSTANTIATE_TK
// Build-trimming switches (plug-ins of user-defined targets are compiled at run time, for one row size):
#ifndef BJX_BUILD_SC
#define BJX_BUILD_SC -1   // -1: every size class; otherwise the one SizeClass to instantiate
#endif
#ifndef BJX_BUILD_DM
#define BJX_BUILD_DM 2    // 0: diagonal metrics only; 1: small dense / low-rank metrics only; 2: both
#endif
#ifndef BJX_BUILD_GEN
#define BJX_BUILD_GEN 2   // 0: velocity Verlet only; 1: general coefficient tables only; 2: both
#endif

// Dynamic shared memory beyond the default 48 KB needs the kernel's opt-in (a host-side attribute call, cheap next to the
// launch; only rows of more than 512 dims ask for it)
template <class K>
static void allow_dynamic_smem(K kern, size_t bytes) {
  if (bytes > 48 * 1024 - 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
}

// A persistent grid over the chains (k_nuts_chains, k_gist_chains, k_ess_chains, k_slice_chains, k_rw_chains), whose warps take the chains from the
// queue dispatch() zeroed: every CTA that stays resident (registers, shared memory) on each SM, at most one per
// kWarpsPerBlock chains.
template <class K, class... Args>
static void launch_persistent(K kern, const LaunchArgs& a, size_t smem, Args... args) {
  allow_dynamic_smem(kern, smem);
  int nb = 1;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kern, kThreads, smem) != cudaSuccess || nb < 1) nb = 1;
  const long long want = ((long long)a.P.C + kWarpsPerBlock - 1) / kWarpsPerBlock;
  const long long ctas = std::min<long long>(want, (long long)sm_count() * nb);
  kern<<<dim3((unsigned)ctas), kThreads, smem, a.stream>>>(args...);
}

template <class R, int TK, bool DM, int KIND>
static int launch_langevin(int kernel_id, const LaunchArgs& a, dim3 grid, size_t smem) {
  if (kernel_id == K_LANGEVIN)
    k_langevin_transition<R, TK, DM, KIND><<<grid, kThreads, smem, a.stream>>>(a.P, a.keys, a.q_in, a.logp_in, a.g_in,
                                                                               a.q_out, a.logp_out, a.g_out, a.langevin);
  else
    k_langevin_chains<R, TK, DM, KIND><<<grid, kThreads, smem, a.stream>>>(a.P, a.q_out, a.logp_out, a.g_out, a.langevin);
  return 0;
}

template <class R, int TK, bool DM, int PRIOR>
static int launch_ess(int kernel_id, const LaunchArgs& a, dim3 grid) {
  const size_t smem = ess_smem_bytes<TK, DM>(a.P.D);
  if (kernel_id == K_ESS) {
    auto kern = k_ess_transition<R, TK, DM, PRIOR>;
    allow_dynamic_smem(kern, smem);
    kern<<<grid, kThreads, smem, a.stream>>>(a.P, a.keys, a.q_in, a.logp_in, a.q_out, a.logp_out, a.ess);
    return 0;
  }
  if constexpr (PRIOR != ESS_PRIOR_NU) {
    launch_persistent(k_ess_chains<R, TK, DM, PRIOR>, a, smem, a.P, a.q_out, a.logp_out, a.ess);
    return 0;
  }
  return -2;
}

// Slice sampling: the warp's rows x and d as elliptical slice sampling's x and nu (ess_smem_bytes)
template <class R, int TK, bool DM>
static int launch_slice(int kernel_id, const LaunchArgs& a, dim3 grid) {
  const size_t smem = ess_smem_bytes<TK, DM>(a.P.D);
  if (kernel_id == K_SLICE) {
    auto kern = k_slice_transition<R, TK, DM>;
    allow_dynamic_smem(kern, smem);
    kern<<<grid, kThreads, smem, a.stream>>>(a.P, a.keys, a.q_in, a.logp_in, a.q_out, a.logp_out, a.slice);
    return 0;
  }
  launch_persistent(k_slice_chains<R, TK, DM>, a, smem, a.P, a.q_out, a.logp_out, a.slice);
  return 0;
}

// Random-walk Metropolis: shared memory only for the target's and the dense sigma's row slices
template <class R, int TK, bool DM>
static int launch_rw(int kernel_id, const LaunchArgs& a, dim3 grid, size_t smem) {
  if (kernel_id == K_RW) {
    k_rw_transition<R, TK, DM><<<grid, kThreads, smem, a.stream>>>(a.P, a.keys, a.q_in, a.logp_in, a.q_out, a.logp_out,
                                                                     a.rw);
    return 0;
  }
  launch_persistent(k_rw_chains<R, TK, DM>, a, smem, a.P, a.q_out, a.logp_out, a.rw);
  return 0;
}

template <class R, int TK, bool DM, bool GEN>
static int launch_gen(int kernel_id, const LaunchArgs& a) {
  const int n_rows = (kernel_id == K_NUTS_DOUBLING) ? a.n_in : a.P.C;
  dim3 grid((n_rows + kWarpsPerBlock - 1) / kWarpsPerBlock), block(kThreads);
  // row count only known on the device: a fixed grid of 6 CTAs per SM strides over the compacted list
  if (kernel_id == K_NUTS_DOUBLING && a.n_in_dev) grid.x = std::min(grid.x, 6u * (unsigned)sm_count());
  size_t smem = needs_row_smem<TK, DM>() ? sizeof(float) * kWarpsPerBlock * a.P.D : 0;
  if (kernel_id == K_NUTS_DOUBLING && a.ckpt_smem) smem += sizeof(float) * kWarpsPerBlock * 2 * a.depth_end * a.P.D;
  cudaStream_t st = a.stream;
  switch (kernel_id) {
    case K_INIT:
      k_init_state<R, TK, DM><<<grid, block, smem, st>>>(a.P, a.q_in, a.logp_out, a.g_out);
      return 0;
    case K_LEAPFROG:
      k_leapfrog<R, TK, DM, GEN><<<grid, block, smem, st>>>(a.P, a.q_out, a.p_io, a.logp_out, a.g_out, a.n);
      return 0;
    case K_HMC:
      k_hmc_transition<R, TK, DM, GEN><<<grid, block, smem, st>>>(a.P, a.keys, a.q_in, a.logp_in, a.g_in, a.q_out,
                                                                   a.logp_out, a.g_out, a.n, a.info);
      return 0;
    case K_MHMC:
      k_mhmc_transition<R, TK, DM, GEN><<<grid, block, smem, st>>>(a.P, a.keys, a.q_in, a.logp_in, a.g_in, a.q_out,
                                                                    a.logp_out, a.g_out, a.n, a.info);
      return 0;
    case K_GHMC:
      k_ghmc_transition<R, TK, DM, GEN><<<grid, block, smem, st>>>(a.P, a.keys, a.q_out, a.logp_out, a.g_out, a.ghmc, a.info);
      return 0;
    case K_MCLMC:  // diagonal metrics only: the host rejects the others before dispatch
      if constexpr (!DM) {
        k_mclmc_transition<R, TK, DM, GEN><<<grid, block, smem, st>>>(a.P, a.keys, a.q_out, a.p_io, a.logp_out, a.g_out,
                                                                       a.mclmc);
        return 0;
      }
      break;
    case K_AMCLMC:  // diagonal metrics only, as K_MCLMC
      if constexpr (!DM) {
        k_amclmc_transition<R, TK, DM, GEN><<<grid, block, smem, st>>>(a.P, a.keys, a.q_in, a.logp_in, a.g_in, a.q_out,
                                                                        a.logp_out, a.g_out, a.amclmc, a.info);
        return 0;
      }
      break;
    case K_MCLMC_TUNE:  // diagonal metrics only, as K_MCLMC
      if constexpr (!DM) {
        k_mclmc_tune<R, TK, DM, GEN><<<grid, block, smem, st>>>(a.P, a.keys, a.q_out, a.p_io, a.logp_out, a.g_out,
                                                                 a.mclmc_tune);
        return 0;
      }
      break;
    case K_AMCLMC_TUNE:  // diagonal metrics only, as K_MCLMC
      if constexpr (!DM) {
        k_amclmc_tune<R, TK, DM, GEN><<<grid, block, smem, st>>>(a.P, a.keys, a.q_out, a.logp_out, a.g_out, a.amclmc_tune);
        return 0;
      }
      break;
    case K_LAPS_BURN_IN:  // diagonal metrics only, as K_MCLMC; a fixed grid and the CTA's sums after the target's rows
      if constexpr (!DM) {
        k_laps_burn_in<R, TK, DM, GEN><<<laps_grid(a.P.C), block, smem + sizeof(float) * (3 * a.P.D + 4), st>>>(
            a.P, a.q_out, a.p_io, a.logp_out, a.g_out, a.laps);
        return 0;
      }
      break;
    case K_GIST: {
      auto kern = k_gist_transition<R, TK, DM, GEN>;
      const size_t gsm = gist_smem_bytes<R, TK, DM>(a.P.D);
      allow_dynamic_smem(kern, gsm);
      kern<<<grid, block, gsm, st>>>(a.P, a.keys, a.q_in, a.logp_in, a.g_in, a.q_out, a.logp_out, a.g_out, a.gist);
      return 0;
    }
    case K_GIST_CHAINS:
      launch_persistent(k_gist_chains<R, TK, DM, GEN>, a, gist_smem_bytes<R, TK, DM>(a.P.D), a.P, a.q_out,
                        a.logp_out, a.g_out, a.gist);
      return 0;
    case K_LANGEVIN:
    case K_LANGEVIN_CHAINS:
      // velocity Verlet instances only (no integrator here); MALA has no metric (dispatched as diagonal), Barker's dense
      // metric exists for dim <= 128
      if constexpr (!GEN && !DM) {
        if (a.langevin.kind == LANGEVIN_MALA) return launch_langevin<R, TK, DM, LANGEVIN_MALA>(kernel_id, a, grid, smem);
        return launch_langevin<R, TK, DM, LANGEVIN_BARKER>(kernel_id, a, grid, smem);
      } else if constexpr (!GEN && R::NS <= 4) {
        if (a.langevin.kind == LANGEVIN_BARKER) return launch_langevin<R, TK, DM, LANGEVIN_BARKER>(kernel_id, a, grid, smem);
      }
      break;
    case K_ESS:
    case K_ESS_CHAINS:
      // velocity Verlet instances only (nothing is integrated); dm selects the small dense prior (dim <= 128), the
      // tensor-core route's nu from HBM exists for the vector rows beyond 128 dims and its loop is a launch per step
      if constexpr (!GEN && !DM) {
        if (a.ess.prior == ESS_PRIOR_DIAG) return launch_ess<R, TK, DM, ESS_PRIOR_DIAG>(kernel_id, a, grid);
        if constexpr (R::VEC && R::NS >= 8) {
          if (a.ess.prior == ESS_PRIOR_NU) return launch_ess<R, TK, DM, ESS_PRIOR_NU>(kernel_id, a, grid);
        }
      } else if constexpr (!GEN && R::NS <= 4) {
        if (a.ess.prior == ESS_PRIOR_DENSE) return launch_ess<R, TK, DM, ESS_PRIOR_DENSE>(kernel_id, a, grid);
      }
      break;
    case K_SLICE:
    case K_SLICE_CHAINS:
      // velocity Verlet instances only (nothing is integrated); dm selects the small dense direction scale (dim <= 128)
      if constexpr (!GEN && (!DM || R::NS <= 4)) return launch_slice<R, TK, DM>(kernel_id, a, grid);
      break;
    case K_RW:
    case K_RW_CHAINS:
      // velocity Verlet instances only (nothing is integrated); dm selects the small dense sigma (dim <= 128)
      if constexpr (!GEN && (!DM || R::NS <= 4)) return launch_rw<R, TK, DM>(kernel_id, a, grid, smem);
      break;
    case K_NUTS_CHAINS:  // the row and the checkpoints of every doubling in shared memory
      launch_persistent(k_nuts_chains<R, TK, DM, GEN>, a,
                        smem + (a.sample.ckpt_smem ? sizeof(float) * kWarpsPerBlock * 2 * a.sample.max_doublings * a.P.D : 0),
                        a.P, a.ws, a.q_out, a.logp_out, a.g_out, a.sample);
      return 0;
    case K_NUTS_DOUBLING:
      if (a.n_in_dev)
        k_nuts_doubling<R, TK, DM, GEN, true><<<grid, block, smem, st>>>(a.P, a.ws, a.depth, a.depth_end, a.n, a.list_in, a.n_in,
                                                                         a.n_in_dev, a.list_out, a.counter, a.q_out, a.logp_out,
                                                                         a.g_out, a.ckpt_smem);
      else
        k_nuts_doubling<R, TK, DM, GEN, false><<<grid, block, smem, st>>>(a.P, a.ws, a.depth, a.depth_end, a.n, a.list_in, a.n_in,
                                                                          nullptr, a.list_out, a.counter, a.q_out, a.logp_out,
                                                                          a.g_out, a.ckpt_smem);
      return 0;
    default:
      break;
  }
  if constexpr (TK == TK_FUNNEL) {  // target-independent kernels are built once, under the funnel launcher
    switch (kernel_id) {
      case K_MOMENTUM:
        k_sample_momentum<R, TK, DM><<<grid, block, smem, st>>>(a.P, a.keys, a.p_io);
        return 0;
      case K_ENERGY:
        k_energy<R, TK, DM><<<grid, block, smem, st>>>(a.P, a.p_io, a.logp_in, a.e_out);
        return 0;
      case K_TURNING:
        k_is_turning<R, TK, DM><<<grid, block, smem, st>>>(a.P, a.pl, a.pr, a.ps, a.out_u8);
        return 0;
      case K_NUTS_INIT:
        k_nuts_init<R, TK, DM><<<grid, block, smem, st>>>(a.P, a.ws, a.keys, a.q_in, a.logp_in, a.g_in, a.q_out,
                                                           a.logp_out, a.g_out, a.mom_override, a.keyint_override,
                                                           a.mom_out);
        return 0;
      default:
        break;
    }
  }
  return -2;
}

template <class R, int TK, bool ALLOW_DM = true>
static int launch_one(int kernel_id, bool dm, const LaunchArgs& a) {
  if (dm) {
    if constexpr (ALLOW_DM && BJX_BUILD_DM != 0) {
      if (a.general_integrator) {
        if constexpr (BJX_BUILD_GEN != 0) return launch_gen<R, TK, true, true>(kernel_id, a);
      } else {
        if constexpr (BJX_BUILD_GEN != 1) return launch_gen<R, TK, true, false>(kernel_id, a);
      }
    }
  } else {
    if constexpr (BJX_BUILD_DM != 1) {
      if (a.general_integrator) {
        if constexpr (BJX_BUILD_GEN != 0) return launch_gen<R, TK, false, true>(kernel_id, a);
      } else {
        if constexpr (BJX_BUILD_GEN != 1) return launch_gen<R, TK, false, false>(kernel_id, a);
      }
    }
  }
  return -2;
}

constexpr bool sc_built(int sc) { return BJX_BUILD_SC < 0 || BJX_BUILD_SC == sc; }

template <int TK>
int Launcher<TK>::launch(int kernel_id, int sc, bool dm, const LaunchArgs& a) {
  constexpr bool small_only = (TK == TK_DENSE || TK == TK_BANANA);
  if constexpr (sc_built(SC_V1)) { if (sc == SC_V1) return launch_one<Row<4, true>, TK>(kernel_id, dm, a); }
  if constexpr (sc_built(SC_S1)) { if (sc == SC_S1) return launch_one<Row<1, false>, TK>(kernel_id, dm, a); }
  if constexpr (sc_built(SC_S4)) { if (sc == SC_S4) return launch_one<Row<4, false>, TK>(kernel_id, dm, a); }
  if constexpr (!small_only) {  // dm beyond 128 dims: the low-rank metric (O(D k) per operation) for rows up to 512
    if constexpr (sc_built(SC_V2)) { if (sc == SC_V2) return launch_one<Row<8, true>, TK>(kernel_id, dm, a); }
    if constexpr (sc_built(SC_V4)) { if (sc == SC_V4) return launch_one<Row<16, true>, TK>(kernel_id, dm, a); }
    if constexpr (sc_built(SC_V8)) { if (sc == SC_V8) return launch_one<Row<32, true>, TK, false>(kernel_id, dm, a); }
  }
  return -2;
}
template struct Launcher<BJX_INSTANTIATE_TK>;
#endif

}  // namespace bjx
