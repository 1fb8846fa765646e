// MALA and Barker entry points of include/bjx.h (blackjax/mcmc/mala.py, blackjax/mcmc/barker.py): one transition and the
// native run loop.  The transition is langevin_transition_row (bjx_kernels.cuh) in k_langevin_transition /
// k_langevin_chains on rows up to 1024 dims, and k_big_langevin (bjx_big.cuh) beyond; initialisation is bjx_init_state.
#include "../../include/bjx.h"
#include "bjx_internal.h"
#include "bjx_big.cuh"
#include "bjx_handle.h"

using namespace bjx;

int bjx_big_langevin(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logp_in, const float* g_in,
                     float* q_out, float* logp_out, float* g_out, float eps, const float* eps_dev, const LangevinArgs& A);

// A configuration the kernels serve, or the reason; sets big when the call takes the CTA-per-chain rows
static int langevin_supported(bjx_handle_t h, int kind, bool& big) {
  const char* name = kind == LANGEVIN_MALA ? "MALA" : "Barker";
  if (kind == LANGEVIN_BARKER) {
    if (h->metric_kind < 0) return bjx_fail(h, BJX_E_STATE, "metric not set: call bjx_set_metric first");
    if (h->metric_kind == BJX_METRIC_DENSE_PER_CHAIN || h->metric_kind == BJX_METRIC_LOW_RANK)
      return bjx_fail(h, BJX_E_UNSUPPORTED, "Barker is built for diagonal, per-chain diagonal and dense (dim <= 128) metrics");
    if (h->metric_kind == BJX_METRIC_DENSE && h->cfg.dim > 128)
      return bjx_fail(h, BJX_E_UNSUPPORTED, "Barker with a dense metric is built for dim <= 128 (not on the tensor-core path)");
  }
  const Route route = kind == LANGEVIN_MALA ? target_route(h) : transition_route(h);
  if (route == ROUTE_DENSE)
    return bjx_fail(h, BJX_E_UNSUPPORTED, std::string(name) + " is not built on the tensor-core dense path (a dense "
                                          "Gaussian target beyond 128 dims)");
  big = route == ROUTE_BIG;
  if (h->cfg.target.kind == BJX_TARGET_USER) {
    auto* pl = static_cast<bjx_plugin_s*>(h->cfg.target.user_plugin);
    if (big ? !pl->launch_big : !pl->launch)
      return bjx_fail(h, BJX_E_UNSUPPORTED, std::string(name) + (big ? " needs a plug-in built with the big-row kernels "
                                                                      "(1024 < dim <= 18432)"
                                                                    : " needs a plug-in built with the row kernels "
                                                                      "(dim <= 1024)"));
  }
  return 0;
}

static int langevin_step(bjx_handle_t h, int kind, const uint32_t* keys, const float* q_in, const float* logp_in,
                         const float* grad_in, float* q_out, float* logp_out, float* grad_out, float step_size,
                         const float* step_size_dev, const bjx_langevin_info* info) {
  const void* ptrs[] = {q_in, grad_in, q_out, grad_out};
  int rc = check_ready(h, false, ptrs, 4);
  if (rc) return rc;
  if (!keys || !logp_in || !logp_out) return bjx_fail(h, BJX_E_INVALID, "bad argument");
  if ((q_in == q_out) != (grad_in == grad_out) || (q_in == q_out) != (logp_in == logp_out))
    return bjx_fail(h, BJX_E_INVALID, "in-place call must alias all of (q, logp, grad)");
  bool big = false;
  if ((rc = langevin_supported(h, kind, big))) return rc;
  LangevinArgs A{};
  A.kind = kind;
  A.chol = h->chol;
  if (info) {
    A.info.acceptance_rate = info->acceptance_rate;
    A.info.is_accepted = info->is_accepted;
    A.info.proposal_position = info->proposal_position;
    A.info.proposal_logdensity = info->proposal_logdensity;
    A.info.proposal_grad = info->proposal_grad;
  }
  if (big)
    return bjx_big_langevin(h, keys, q_in, logp_in, grad_in, q_out, logp_out, grad_out, step_size, step_size_dev, A);
  LaunchArgs a{};
  a.P = make_params(h, step_size, step_size_dev);
  a.keys = keys;
  a.q_in = q_in;
  a.logp_in = logp_in;
  a.g_in = grad_in;
  a.q_out = q_out;
  a.logp_out = logp_out;
  a.g_out = grad_out;
  a.langevin = A;
  return dispatch(h, K_LANGEVIN, true, a);
}

static int langevin_sample(bjx_handle_t h, int kind, const uint32_t* rng_key, float* q, float* logp, float* grad,
                           float step_size, const float* step_size_dev, int32_t num_steps, float* history, int32_t thin,
                           float* acceptance_history) {
  const void* ptrs[] = {q, grad};
  int rc = check_ready(h, false, ptrs, 2);
  if (rc) return rc;
  if (!rng_key || !logp || num_steps < 0 || thin < 1) return bjx_fail(h, BJX_E_INVALID, "bad argument");
  bool big = false;
  if ((rc = langevin_supported(h, kind, big))) return rc;
  if (num_steps == 0) return 0;
  return run_loop(h, rng_key, num_steps, history, thin, [&](const RunLoop& loop) {
    LangevinArgs A{};
    A.kind = kind;
    A.chol = h->chol;
    A.loop = loop;
    A.acceptance_history = acceptance_history;
    if (big) return bjx_big_langevin(h, nullptr, q, logp, grad, q, logp, grad, step_size, step_size_dev, A);
    LaunchArgs a{};
    a.P = make_params(h, step_size, step_size_dev);
    a.q_out = q;
    a.logp_out = logp;
    a.g_out = grad;
    a.langevin = A;
    return dispatch(h, K_LANGEVIN_CHAINS, true, a);
  });
}

extern "C" int bjx_mala_step(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logp_in,
                             const float* grad_in, float* q_out, float* logp_out, float* grad_out, float step_size,
                             const float* step_size_dev, const bjx_langevin_info* info) {
  return langevin_step(h, LANGEVIN_MALA, keys, q_in, logp_in, grad_in, q_out, logp_out, grad_out, step_size,
                       step_size_dev, info);
}

extern "C" int bjx_barker_step(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logp_in,
                               const float* grad_in, float* q_out, float* logp_out, float* grad_out, float step_size,
                               const float* step_size_dev, const bjx_langevin_info* info) {
  return langevin_step(h, LANGEVIN_BARKER, keys, q_in, logp_in, grad_in, q_out, logp_out, grad_out, step_size,
                       step_size_dev, info);
}

extern "C" int bjx_mala_sample(bjx_handle_t h, const uint32_t* rng_key, float* q, float* logp, float* grad, float step_size,
                               const float* step_size_dev, int32_t num_steps, float* history, int32_t thin,
                               float* acceptance_history) {
  return langevin_sample(h, LANGEVIN_MALA, rng_key, q, logp, grad, step_size, step_size_dev, num_steps, history, thin,
                         acceptance_history);
}

extern "C" int bjx_barker_sample(bjx_handle_t h, const uint32_t* rng_key, float* q, float* logp, float* grad,
                                 float step_size, const float* step_size_dev, int32_t num_steps, float* history,
                                 int32_t thin, float* acceptance_history) {
  return langevin_sample(h, LANGEVIN_BARKER, rng_key, q, logp, grad, step_size, step_size_dev, num_steps, history, thin,
                         acceptance_history);
}
