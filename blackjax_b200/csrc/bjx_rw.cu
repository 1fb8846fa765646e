// Random-walk Metropolis entry points of include/bjx.h (blackjax/mcmc/random_walk.py: the additive step, rmh and
// irmh): the Gaussian proposal, one transition and the native run loop.  The transition is rw_transition_row
// (bjx_kernels.cuh) in k_rw_transition / k_rw_chains on rows up to 1024 dims, and k_big_rw (bjx_big.cuh) beyond;
// initialisation is bjx_init_state.  Two routes, chosen from the handle as slice sampling's are (bjx_slice.cu):
//   rows, [D] sigma or [D, D] sigma at dim <= 128: the state in registers, the native loop one persistent launch;
//   big rows (1024 < dim <= 18432), [D] sigma: one CTA per chain, the proposal in shared memory.
#include "../../include/bjx.h"
#include "bjx_internal.h"
#include "bjx_big.cuh"
#include "bjx_handle.h"

using namespace bjx;

int bjx_big_rw(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logp_in, float* q_out,
               float* logp_out, const RwArgs& A);

// 1 / sigma, elementwise
static __global__ void k_rw_reciprocal(const float* __restrict__ s, float* __restrict__ r, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) r[i] = 1.0f / s[i];
}

extern "C" int bjx_set_rw_proposal(bjx_handle_t h, int32_t kind, const float* mean, int32_t sigma_kind,
                                   const float* sigma) {
  if (!h || !sigma) return bjx_fail(h, BJX_E_INVALID, "null argument");
  if (kind != BJX_RW_ADDITIVE && kind != BJX_RW_INDEPENDENT)
    return bjx_fail(h, BJX_E_INVALID, "kind must be BJX_RW_ADDITIVE or BJX_RW_INDEPENDENT");
  if (kind == BJX_RW_INDEPENDENT && !mean)
    return bjx_fail(h, BJX_E_INVALID, "a position-independent proposal needs its mean");
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  int rc = bjx_store_scale(h, sigma_kind, sigma, h->rw_sigma, h->rw_sigma_cap, "random-walk sigma");
  if (rc) return rc;
  if (kind == BJX_RW_INDEPENDENT) {
    const int D = h->cfg.dim;
    if ((rc = bjx_grow(h, h->rw_mean, h->rw_mean_cap, 2 * (size_t)D, sizeof(float)))) return rc;
    BJX_CUDA(cudaMemcpyAsync(h->rw_mean, mean, D * sizeof(float), cudaMemcpyDeviceToDevice, h->stream));
    if (sigma_kind == BJX_METRIC_DIAG) {
      k_rw_reciprocal<<<(D + 255) / 256, 256, 0, h->stream>>>(h->rw_sigma, h->rw_mean + D, D);
      BJX_CHECK_LAUNCH("k_rw_reciprocal");
    }
  }
  h->rw_kind = kind;
  h->rw_sigma_kind = sigma_kind;
  return 0;
}

// The route of a call, or the reason it has none: sets big
static int rw_route(bjx_handle_t h, int32_t correct, bool& big) {
  if (h->rw_kind < 0)
    return bjx_fail(h, BJX_E_UNSUPPORTED, "random-walk Metropolis needs a proposal: call bjx_set_rw_proposal first");
  if (target_route(h) == ROUTE_DENSE)
    return bjx_fail(h, BJX_E_UNSUPPORTED, "random-walk Metropolis is not built on the tensor-core dense target path (a "
                                          "dense Gaussian target beyond 128 dims)");
  big = h->sc == SC_BIG;
  if (h->cfg.target.kind == BJX_TARGET_USER) {
    auto* pl = static_cast<bjx_plugin_s*>(h->cfg.target.user_plugin);
    if (big ? !pl->launch_big : !pl->launch)
      return bjx_fail(h, BJX_E_UNSUPPORTED, big ? "random-walk Metropolis needs a plug-in built with the big-row kernels "
                                                  "(1024 < dim <= 18432)"
                                                : "random-walk Metropolis needs a plug-in built with the row kernels "
                                                  "(dim <= 1024)");
  }
  if (correct && h->rw_kind != BJX_RW_INDEPENDENT)
    return bjx_fail(h, BJX_E_UNSUPPORTED, "the proposal correction is built for a position-independent proposal "
                                          "(BJX_RW_INDEPENDENT) only");
  if (correct && h->rw_sigma_kind == BJX_METRIC_DENSE)
    return bjx_fail(h, BJX_E_UNSUPPORTED, "the proposal correction is not built for a dense sigma");
  return 0;
}

static RwArgs rw_args(bjx_handle_t h, int32_t correct) {
  RwArgs A{};
  A.kind = h->rw_kind;
  A.mean = h->rw_kind == BJX_RW_INDEPENDENT ? h->rw_mean : nullptr;
  A.sigma = h->rw_sigma;
  A.inv_sigma = h->rw_kind == BJX_RW_INDEPENDENT ? h->rw_mean + h->cfg.dim : nullptr;
  A.correct = correct != 0;
  return A;
}

extern "C" int bjx_rw_step(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logp_in, float* q_out,
                           float* logp_out, int32_t correct, const bjx_rw_info* info) {
  const void* ptrs[] = {q_in, q_out};
  int rc = check_ready(h, false, ptrs, 2);
  if (rc) return rc;
  if (!keys || !logp_in || !logp_out) return bjx_fail(h, BJX_E_INVALID, "bad argument");
  if ((q_in == q_out) != (logp_in == logp_out))
    return bjx_fail(h, BJX_E_INVALID, "in-place call must alias both of (q, logp)");
  bool big = false;
  if ((rc = rw_route(h, correct, big))) return rc;
  RwArgs A = rw_args(h, correct);
  if (info) {
    A.info.acceptance_rate = info->acceptance_rate;
    A.info.is_accepted = info->is_accepted;
  }
  if (big) return bjx_big_rw(h, keys, q_in, logp_in, q_out, logp_out, A);
  LaunchArgs a{};
  a.P = make_params(h, 0.f, nullptr);
  a.keys = keys;
  a.q_in = q_in;
  a.logp_in = logp_in;
  a.q_out = q_out;
  a.logp_out = logp_out;
  a.rw = A;
  return dispatch(h, K_RW, true, a);
}

extern "C" int bjx_rw_sample(bjx_handle_t h, const uint32_t* rng_key, float* q, float* logp, int32_t num_steps,
                             int32_t correct, float* history, int32_t thin, float* acceptance_history) {
  const void* ptrs[] = {q};
  int rc = check_ready(h, false, ptrs, 1);
  if (rc) return rc;
  if (!rng_key || !logp || num_steps < 0 || thin < 1) return bjx_fail(h, BJX_E_INVALID, "bad argument");
  bool big = false;
  if ((rc = rw_route(h, correct, big))) return rc;
  if (num_steps == 0) return 0;
  return run_loop(h, rng_key, num_steps, history, thin, [&](const RunLoop& loop) {
    RwArgs A = rw_args(h, correct);
    A.loop = loop;
    A.acceptance_history = acceptance_history;
    if (big) return bjx_big_rw(h, nullptr, q, logp, q, logp, A);
    LaunchArgs a{};
    a.P = make_params(h, 0.f, nullptr);
    a.q_out = q;
    a.logp_out = logp;
    a.rw = A;
    return dispatch(h, K_RW_CHAINS, true, a);
  });
}
