// Elliptical slice sampling entry points of include/bjx.h (blackjax/mcmc/elliptical_slice.py): the prior, one transition
// and the native run loop.  The transition is ess_transition_row (bjx_kernels.cuh) in k_ess_transition / k_ess_chains on
// rows up to 1024 dims, and k_big_ess (bjx_big.cuh) beyond; initialisation is bjx_init_state.  Three routes, chosen from
// the handle:
//   rows, diagonal prior or dense prior at dim <= 128: nu is drawn in the warp (the dense one with the small matvec), and
//     the native loop is one persistent launch;
//   rows, dense prior at 128 < dim <= 1024: L z is one float32-accurate tensor-core product per transition
//     (bjx_dense_prior_product), which the warp kernel reads; the native loop is three launches per transition;
//   big rows (1024 < dim <= 18432), diagonal prior: one CTA per chain, nu in a [C, D] scratch.
#include <math.h>

#include <vector>

#include "../../include/bjx.h"
#include "bjx_internal.h"
#include "bjx_big.cuh"
#include "bjx_handle.h"

using namespace bjx;

int bjx_big_ess(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logl_in, float* q_out,
                float* logl_out, const EssArgs& A);
int bjx_dense_prior_product(bjx_handle_t h, const uint32_t* keys, const float** lz);

extern "C" int bjx_set_elliptical_prior(bjx_handle_t h, int32_t kind, const float* mean, const float* cov) {
  if (!h || !mean || !cov) return bjx_fail(h, BJX_E_INVALID, "null argument");
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  const int D = h->cfg.dim;
  size_t elems;
  if (kind == BJX_METRIC_DIAG) {
    elems = D;
  } else if (kind == BJX_METRIC_DENSE) {
    if (D > 1024) return bjx_fail(h, BJX_E_UNSUPPORTED, "a dense elliptical slice prior is built for dim <= 1024");
    if (D > 128 && D % 4 != 0)
      return bjx_fail(h, BJX_E_UNSUPPORTED, "a dense elliptical slice prior with dim > 128 needs dim % 4 == 0 "
                                            "(tensor-core product)");
    elems = (size_t)D * D;
  } else {
    return bjx_fail(h, BJX_E_INVALID, "The covariance matrix has the wrong number of dimensions: expected 1 or 2");
  }
  std::vector<float> buf((size_t)D + elems), c(elems);
  BJX_CUDA(cudaMemcpyAsync(buf.data(), mean, (size_t)D * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  BJX_CUDA(cudaMemcpyAsync(c.data(), cov, elems * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  BJX_CUDA(cudaStreamSynchronize(h->stream));
  if (kind == BJX_METRIC_DIAG) {
    for (int i = 0; i < D; ++i) buf[(size_t)D + i] = sqrtf(c[i]);  // elliptical_slice.py:95
  } else {
    std::vector<double> L;  // elliptical_slice.py:98, formed in float64 as bjx_set_metric does
    if (!cholesky_f64(c, D, L)) return bjx_fail(h, BJX_E_INVALID, "prior covariance matrix is not positive definite");
    for (size_t k = 0; k < elems; ++k) buf[(size_t)D + k] = (float)L[k];
  }
  int rc = bjx_grow(h, h->ess_prior, h->ess_prior_cap, buf.size(), sizeof(float));
  if (rc) return rc;
  BJX_CUDA(cudaMemcpyAsync(h->ess_prior, buf.data(), buf.size() * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  BJX_CUDA(cudaStreamSynchronize(h->stream));
  h->ess_kind = kind;
  h->dense_version++;  // the tensor-core route re-splits L
  return 0;
}

// The route of a call, or the reason it has none: sets prior (EssPrior) and big
static int ess_route(bjx_handle_t h, int& prior, bool& big) {
  if (h->ess_kind < 0)
    return bjx_fail(h, BJX_E_UNSUPPORTED, "elliptical slice sampling needs a prior: call bjx_set_elliptical_prior first");
  if (target_route(h) == ROUTE_DENSE)
    return bjx_fail(h, BJX_E_UNSUPPORTED, "elliptical slice sampling is not built on the tensor-core dense target path "
                                          "(a dense Gaussian target beyond 128 dims)");
  big = h->sc == SC_BIG;
  if (h->ess_kind == BJX_METRIC_DIAG) prior = ESS_PRIOR_DIAG;
  else prior = h->cfg.dim <= 128 ? ESS_PRIOR_DENSE : ESS_PRIOR_NU;
  if (h->cfg.target.kind == BJX_TARGET_USER) {
    auto* pl = static_cast<bjx_plugin_s*>(h->cfg.target.user_plugin);
    if (big ? !pl->launch_big : !pl->launch)
      return bjx_fail(h, BJX_E_UNSUPPORTED, big ? "elliptical slice sampling needs a plug-in built with the big-row "
                                                  "kernels (1024 < dim <= 18432)"
                                                : "elliptical slice sampling needs a plug-in built with the row kernels "
                                                  "(dim <= 1024)");
  }
  return 0;
}

// The arguments every launch shares, with the handle's scratch: nu [C, D] on the big rows
static int ess_args(bjx_handle_t h, int prior, bool big, int max_subiter, EssArgs& A) {
  const size_t rows = big ? (size_t)h->cfg.n_chains * h->cfg.dim : 0;
  int rc = bjx_grow(h, h->ess_ws, h->ess_ws_cap, rows, sizeof(float));
  if (rc) return rc;
  A = EssArgs{};
  A.prior = prior;
  A.mean = h->ess_prior;
  A.scale = h->ess_prior + h->cfg.dim;
  A.nu = big ? h->ess_ws : nullptr;
  A.max_subiter = max_subiter;
  return 0;
}

extern "C" int bjx_elliptical_slice_step(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logl_in,
                                         float* q_out, float* logl_out, int32_t max_subiter,
                                         const bjx_elliptical_slice_info* info) {
  const void* ptrs[] = {q_in, q_out, info && info->momentum ? info->momentum : q_in};
  int rc = check_ready(h, false, ptrs, 3);
  if (rc) return rc;
  if (!keys || !logl_in || !logl_out || max_subiter < 1) return bjx_fail(h, BJX_E_INVALID, "bad argument");
  if ((q_in == q_out) != (logl_in == logl_out))
    return bjx_fail(h, BJX_E_INVALID, "in-place call must alias both of (q, logl)");
  int prior = 0;
  bool big = false;
  if ((rc = ess_route(h, prior, big))) return rc;
  EssArgs A;
  if ((rc = ess_args(h, prior, big, max_subiter, A))) return rc;
  if (info) {
    A.info.momentum = info->momentum;
    A.info.theta = info->theta;
    A.info.subiter = info->subiter;
    A.info.exhausted = info->exhausted;
  }
  if (big) return bjx_big_ess(h, keys, q_in, logl_in, q_out, logl_out, A);
  if (prior == ESS_PRIOR_NU) {
    const float* lz = nullptr;
    if ((rc = bjx_dense_prior_product(h, keys, &lz))) return rc;
    A.nu = const_cast<float*>(lz);
  }
  LaunchArgs a{};
  a.P = make_params(h, 0.f, nullptr);
  a.keys = keys;
  a.q_in = q_in;
  a.logp_in = logl_in;
  a.q_out = q_out;
  a.logp_out = logl_out;
  a.ess = A;
  return dispatch(h, K_ESS, true, a);
}

extern "C" int bjx_elliptical_slice_sample(bjx_handle_t h, const uint32_t* rng_key, float* q, float* logl,
                                           int32_t num_steps, int32_t max_subiter, float* history, int32_t thin,
                                           int32_t* subiter_history) {
  const void* ptrs[] = {q};
  int rc = check_ready(h, false, ptrs, 1);
  if (rc) return rc;
  if (!rng_key || !logl || num_steps < 0 || thin < 1 || max_subiter < 1)
    return bjx_fail(h, BJX_E_INVALID, "bad argument");
  int prior = 0;
  bool big = false;
  if ((rc = ess_route(h, prior, big))) return rc;
  if (num_steps == 0) return 0;
  if (prior == ESS_PRIOR_NU)  // per transition: the normal draw, the product and the slice kernel, all enqueued
    return run_steps(h, rng_key, num_steps, history, thin, q, [&](int t, const uint32_t* key_t) {
      bjx_elliptical_slice_info info{};
      info.subiter = step_row(subiter_history, t, h->cfg.n_chains);
      return bjx_elliptical_slice_step(h, key_t, q, logl, q, logl, max_subiter, &info);
    });
  return run_loop(h, rng_key, num_steps, history, thin, [&](const RunLoop& loop) {
    EssArgs A;
    int rc = ess_args(h, prior, big, max_subiter, A);
    if (rc) return rc;
    A.loop = loop;
    A.subiter_history = subiter_history;
    if (big) return bjx_big_ess(h, nullptr, q, logl, q, logl, A);
    LaunchArgs a{};
    a.P = make_params(h, 0.f, nullptr);
    a.q_out = q;
    a.logp_out = logl;
    a.ess = A;
    return dispatch(h, K_ESS_CHAINS, true, a);
  });
}
