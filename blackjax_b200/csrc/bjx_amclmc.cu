// Adjusted MCLMC (MAMS) entry points of include/bjx.h (blackjax/mcmc/adjusted_mclmc.py, adjusted_mclmc_dynamic.py): one
// transition and the native run loop.  The transition itself is k_amclmc_transition (bjx_kernels.cuh), instantiated per
// target by bjx_launch.cuh; initialisation is bjx_init_state (adjusted_mclmc.init is value_and_grad).
#include "../../include/bjx.h"
#include "bjx_internal.h"
#include "bjx_launch.cuh"
#include "bjx_handle.h"

using namespace bjx;

static int amclmc_transition(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logp_in,
                             const float* grad_in, float* q_out, float* logp_out, float* grad_out, float step_size,
                             const float* step_size_dev, const AmclmcArgs& A, const bjx_info* info) {
  const void* ptrs[] = {q_in, grad_in, q_out, grad_out};
  int rc = check_ready(h, true, ptrs, 4);
  if (rc) return rc;
  if (!keys || !logp_in || !logp_out || A.n < 0) return bjx_fail(h, BJX_E_INVALID, "bad argument");
  if ((q_in == q_out) != (grad_in == grad_out) || (q_in == q_out) != (logp_in == logp_out))
    return bjx_fail(h, BJX_E_INVALID, "in-place call must alias all of (q, logp, grad)");
  if ((rc = mclmc_transition_supported(h, "adjusted MCLMC"))) return rc;
  LaunchArgs a{};
  a.P = make_params(h, step_size, step_size_dev);
  a.keys = keys;
  a.q_in = q_in;
  a.logp_in = logp_in;
  a.g_in = grad_in;
  a.q_out = q_out;
  a.logp_out = logp_out;
  a.g_out = grad_out;
  a.amclmc = A;
  a.amclmc.avg = h->steps_avg;
  if (info) {
    a.info.acceptance_rate = info->acceptance_rate;
    a.info.is_accepted = info->is_accepted;
    a.info.is_divergent = info->is_divergent;
    a.info.energy = info->energy;
    a.info.num_integration_steps = info->num_integration_steps;
    a.info.momentum = info->momentum;
    a.info.proposal_position = info->proposal_position;
    a.info.proposal_momentum = info->proposal_momentum;
  }
  return dispatch(h, K_AMCLMC, true, a);
}

extern "C" int bjx_adjusted_mclmc_step(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logp_in,
                                       const float* grad_in, float* q_out, float* logp_out, float* grad_out,
                                       float step_size, const float* step_size_dev, int32_t num_integration_steps,
                                       float L_proposal_factor, const bjx_info* info) {
  AmclmcArgs A{};
  A.L_factor = L_proposal_factor;
  A.n = num_integration_steps;
  A.rule = AMCLMC_STEPS_FIXED;
  return amclmc_transition(h, keys, q_in, logp_in, grad_in, q_out, logp_out, grad_out, step_size, step_size_dev, A, info);
}

extern "C" int bjx_adjusted_mclmc_sample(bjx_handle_t h, const uint32_t* rng_key, float* q, float* logp, float* grad,
                                         float step_size, const float* step_size_dev, float L_proposal_factor,
                                         int32_t steps_rule, int32_t num_integration_steps, float steps_scale,
                                         int32_t min_steps, uint32_t* random_generator_arg, int32_t num_steps,
                                         float* history, int32_t thin, float* acceptance_history,
                                         int32_t* steps_history) {
  if (!h || !rng_key || num_steps < 0 || thin < 1) return bjx_fail(h, BJX_E_INVALID, "bad argument");
  if (steps_rule < BJX_AMCLMC_STEPS_FIXED || steps_rule > BJX_AMCLMC_STEPS_UNIFORM)
    return bjx_fail(h, BJX_E_INVALID, "unknown steps_rule");
  if (steps_rule != BJX_AMCLMC_STEPS_FIXED && !random_generator_arg)
    return bjx_fail(h, BJX_E_INVALID, "the dynamic step-count rules need random_generator_arg");
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  if (num_steps == 0) return 0;
  AmclmcArgs A{};
  A.L_factor = L_proposal_factor;
  A.n = num_integration_steps;
  A.rule = steps_rule;
  A.min_steps = min_steps;
  A.scale = steps_scale;
  A.rga = random_generator_arg;
  const int C = h->cfg.n_chains;
  return run_steps(h, rng_key, num_steps, history, thin, q, [&](int t, const uint32_t* key_t) {
    bjx_info info{};
    info.acceptance_rate = step_row(acceptance_history, t, C);
    info.num_integration_steps = step_row(steps_history, t, C);
    return amclmc_transition(h, key_t, q, logp, grad, q, logp, grad, step_size, step_size_dev, A, &info);
  });
}
