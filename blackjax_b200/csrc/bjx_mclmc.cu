// MCLMC entry points of include/bjx.h (blackjax/mcmc/mclmc.py): init, one transition, and the native run loop.  The
// transition itself is k_mclmc_transition (bjx_kernels.cuh), instantiated per target by bjx_launch.cuh.
#include "../../include/bjx.h"
#include "bjx_internal.h"
#include "bjx_launch.cuh"
#include "bjx_handle.h"

using namespace bjx;

// generate_unit_vector (util.py:94-113) for every chain: one warp per chain, any dim
static __global__ void k_unit_vector(Params P, const uint32_t* __restrict__ keys, float* __restrict__ p_out) {
  const int lane = threadIdx.x & 31;
  const int chain = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (chain >= P.C) return;
  const Key k = chain_key(P, keys, chain);
  float* row = p_out + (size_t)chain * P.D;
  float ss = 0.f;
  for (int e = lane; e < P.D; e += 32) {
    const float z = normal_at(k, (uint32_t)e);
    row[e] = z;
    ss = __fmaf_rn(z, z, ss);
  }
  const float n = sqrtf(warp_sum(ss));
  for (int e = lane; e < P.D; e += 32) row[e] = __fdiv_rn(row[e], n);
}

// The dimensions the MCLMC kernels are built for; BJX_E_UNSUPPORTED with the reason otherwise.
static int mclmc_supported(bjx_handle_t h, const std::string& name = "MCLMC") {
  if (h->cfg.dim < 2)
    return bjx_fail(h, BJX_E_UNSUPPORTED, name + " needs dim >= 2 (the target distribution must have more than 1 dimension)");
  return 0;
}

int mclmc_transition_supported(bjx_handle_t h, const char* name) {
  const std::string n(name);
  int rc = mclmc_supported(h, n);
  if (rc) return rc;
  if (h->metric_kind != BJX_METRIC_DIAG && h->metric_kind != BJX_METRIC_DIAG_PER_CHAIN)
    return bjx_fail(h, BJX_E_UNSUPPORTED, n + " is built for diagonal metrics ([dim] or per-chain [n_chains, dim])");
  switch (transition_route(h)) {
    case ROUTE_DENSE: return bjx_fail(h, BJX_E_UNSUPPORTED, n + " with a dense Gaussian target is built for dim <= 128");
    case ROUTE_BIG: return bjx_fail(h, BJX_E_UNSUPPORTED, n + " is built for dim <= 1024 (the warp-per-chain kernels)");
    case ROUTE_ROWS: break;
  }
  return 0;
}

extern "C" int bjx_mclmc_init(bjx_handle_t h, const uint32_t* keys, const float* q, float* logp_out, float* grad_out,
                              float* p_out) {
  const void* ptrs[] = {q, grad_out, p_out};
  int rc = check_ready(h, false, ptrs, 3);
  if (rc) return rc;
  if (!keys || !logp_out) return bjx_fail(h, BJX_E_INVALID, "null argument");
  if ((rc = mclmc_supported(h))) return rc;
  if ((rc = bjx_init_state(h, q, logp_out, grad_out))) return rc;
  const Params P = make_params(h, 0.f, nullptr);
  k_unit_vector<<<(P.C + kWarpsPerBlock - 1) / kWarpsPerBlock, kThreads, 0, h->stream>>>(P, keys, p_out);
  BJX_CHECK_LAUNCH("k_unit_vector");
  return 0;
}

extern "C" int bjx_mclmc_step(bjx_handle_t h, const uint32_t* keys, float* q, float* p, float* logp, float* grad,
                              float step_size, const float* step_size_dev, float L, const float* L_dev, float energy_cutoff,
                              const bjx_mclmc_info* info) {
  const void* ptrs[] = {q, p, grad};
  int rc = check_ready(h, true, ptrs, 3);
  if (rc) return rc;
  if (!keys || !logp) return bjx_fail(h, BJX_E_INVALID, "null argument");
  if ((rc = mclmc_transition_supported(h, "MCLMC"))) return rc;
  LaunchArgs a{};
  a.P = make_params(h, step_size, step_size_dev);
  a.keys = keys;
  a.q_out = q;
  a.p_io = p;
  a.logp_out = logp;
  a.g_out = grad;
  a.mclmc.L = L;
  a.mclmc.L_dev = L_dev;
  a.mclmc.energy_cutoff = energy_cutoff;
  if (info) {
    a.mclmc.kinetic_change = info->kinetic_change;
    a.mclmc.energy_change = info->energy_change;
    a.mclmc.nonans = info->nonans;
  }
  return dispatch(h, K_MCLMC, true, a);
}

extern "C" int bjx_mclmc_sample(bjx_handle_t h, const uint32_t* rng_key, float* q, float* p, float* logp, float* grad,
                                float step_size, const float* step_size_dev, float L, const float* L_dev, float energy_cutoff,
                                int32_t num_steps, float* history, int32_t thin, float* energy_change_history) {
  if (!h || !rng_key || num_steps < 0 || thin < 1) return bjx_fail(h, BJX_E_INVALID, "bad argument");
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  if (num_steps == 0) return 0;
  return run_steps(h, rng_key, num_steps, history, thin, q, [&](int t, const uint32_t* key_t) {
    bjx_mclmc_info info{};
    info.energy_change = step_row(energy_change_history, t, h->cfg.n_chains);
    return bjx_mclmc_step(h, key_t, q, p, logp, grad, step_size, step_size_dev, L, L_dev, energy_cutoff, &info);
  });
}
