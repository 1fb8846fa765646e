// GIST entry points of include/bjx.h (blackjax/mcmc/composed: gist_trajectory_length, gist_step_size): one transition and
// the native run loop.  The transition is gist_transition_row (bjx_kernels.cuh) in k_gist_transition / k_gist_chains,
// instantiated per target by bjx_launch.cuh; initialisation is bjx_init_state (the seam's init is hmc.init).
#include "../../include/bjx.h"
#include "bjx_internal.h"
#include "bjx_launch.cuh"
#include "bjx_handle.h"

using namespace bjx;

// Parameters in range and a configuration the row kernels serve, or the reason
static int gist_supported(bjx_handle_t h, const bjx_gist_params* prm) {
  if (!prm) return bjx_fail(h, BJX_E_INVALID, "null params");
  if (prm->instance == BJX_GIST_TRAJECTORY_LENGTH) {
    if (prm->max_num_steps < 1) return bjx_fail(h, BJX_E_INVALID, "GIST: max_num_steps must be >= 1");
    if (!(prm->path_fraction >= 0.f && prm->path_fraction <= 1.f))
      return bjx_fail(h, BJX_E_INVALID, "GIST: path_fraction must lie in [0, 1]");
  } else if (prm->instance == BJX_GIST_STEP_SIZE) {
    if (prm->num_integration_steps < 1) return bjx_fail(h, BJX_E_INVALID, "GIST: num_integration_steps must be >= 1");
    if (prm->max_search_steps < 0) return bjx_fail(h, BJX_E_INVALID, "GIST: max_search_steps must be >= 0");
    if (prm->criterion != BJX_GIST_SYMMETRIC && prm->criterion != BJX_GIST_ASYMMETRIC)
      return bjx_fail(h, BJX_E_INVALID, "GIST: criterion must be BJX_GIST_SYMMETRIC or BJX_GIST_ASYMMETRIC");
  } else {
    return bjx_fail(h, BJX_E_INVALID, "GIST: unknown instance");
  }
  switch (transition_route(h)) {
    case ROUTE_BIG: return bjx_fail(h, BJX_E_UNSUPPORTED, "GIST is built for dim <= 1024 (the warp-per-chain kernels)");
    case ROUTE_DENSE:
      return bjx_fail(h, BJX_E_UNSUPPORTED, "GIST is not built on the tensor-core dense path (a dense metric or a dense "
                                            "Gaussian target beyond 128 dims)");
    case ROUTE_ROWS: break;
  }
  if (h->cfg.target.kind == BJX_TARGET_USER && !static_cast<bjx_plugin_s*>(h->cfg.target.user_plugin)->launch)
    return bjx_fail(h, BJX_E_UNSUPPORTED, "GIST needs a plug-in built with the row kernels (dim <= 1024)");
  return 0;
}

// The launch arguments shared by both entry points, with the handle's scratch (4 rows [C,D])
static int gist_args(bjx_handle_t h, const bjx_gist_params* prm, float step_size, const float* step_size_dev, LaunchArgs& a) {
  const size_t rows = (size_t)4 * h->cfg.n_chains * h->cfg.dim;
  int rc = bjx_grow(h, h->gist_ws, h->gist_ws_cap, rows, sizeof(float));
  if (rc) return rc;
  a.P = make_params(h, step_size, step_size_dev);
  a.gist.instance = prm->instance;
  a.gist.path_fraction = prm->path_fraction;
  a.gist.max_num_steps = prm->max_num_steps;
  a.gist.n_int = prm->num_integration_steps;
  a.gist.max_search_steps = prm->max_search_steps;
  a.gist.asymmetric = prm->criterion == BJX_GIST_ASYMMETRIC;
  a.gist.ws = h->gist_ws;
  return 0;
}

extern "C" int bjx_gist_step(bjx_handle_t h, const bjx_gist_params* params, const uint32_t* keys, const float* q_in,
                             const float* logp_in, const float* grad_in, float* q_out, float* logp_out, float* grad_out,
                             float step_size, const float* step_size_dev, const bjx_gist_info* info) {
  const void* ptrs[] = {q_in, grad_in, q_out, grad_out};
  int rc = check_ready(h, true, ptrs, 4);
  if (rc) return rc;
  if (!keys || !logp_in || !logp_out) return bjx_fail(h, BJX_E_INVALID, "bad argument");
  if ((q_in == q_out) != (grad_in == grad_out) || (q_in == q_out) != (logp_in == logp_out))
    return bjx_fail(h, BJX_E_INVALID, "in-place call must alias all of (q, logp, grad)");
  if ((rc = gist_supported(h, params))) return rc;
  LaunchArgs a{};
  if ((rc = gist_args(h, params, step_size, step_size_dev, a))) return rc;
  a.keys = keys;
  a.q_in = q_in;
  a.logp_in = logp_in;
  a.g_in = grad_in;
  a.q_out = q_out;
  a.logp_out = logp_out;
  a.g_out = grad_out;
  if (info) {
    GistInfoPtrs& o = a.gist.info;
    o.acceptance_rate = info->acceptance_rate;
    o.is_accepted = info->is_accepted;
    o.is_divergent = info->is_divergent;
    o.energy = info->energy;
    o.momentum = info->momentum;
    o.num_integration_steps = info->num_integration_steps;
    o.forward = info->forward;
    o.reverse = info->reverse;
    o.rejected = info->rejected;
    o.a = info->a;
    o.b = info->b;
    o.step_size = info->step_size;
  }
  return dispatch(h, K_GIST, true, a);
}

extern "C" int bjx_gist_sample(bjx_handle_t h, const bjx_gist_params* params, const uint32_t* rng_key, float* q, float* logp,
                               float* grad, float step_size, const float* step_size_dev, int32_t num_steps, float* history,
                               int32_t thin, float* acceptance_history, int32_t* num_integration_steps_history) {
  const void* ptrs[] = {q, grad};
  int rc = check_ready(h, true, ptrs, 2);
  if (rc) return rc;
  if (!rng_key || !logp || num_steps < 0 || thin < 1) return bjx_fail(h, BJX_E_INVALID, "bad argument");
  if ((rc = gist_supported(h, params))) return rc;
  if (num_steps == 0) return 0;
  return run_loop(h, rng_key, num_steps, history, thin, [&](const RunLoop& loop) {
    LaunchArgs a{};
    int rc = gist_args(h, params, step_size, step_size_dev, a);
    if (rc) return rc;
    a.q_out = q;
    a.logp_out = logp;
    a.g_out = grad;
    a.gist.loop = loop;
    a.gist.acceptance_history = acceptance_history;
    a.gist.nint_history = num_integration_steps_history;
    return dispatch(h, K_GIST_CHAINS, true, a);
  });
}
