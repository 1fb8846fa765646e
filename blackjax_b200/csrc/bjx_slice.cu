// Slice sampling entry points of include/bjx.h (blackjax/mcmc/slice.py, the multivariate slice sampler): the direction
// scale, one transition and the native run loop.  The transition is slice_transition_row (bjx_kernels.cuh) in
// k_slice_transition / k_slice_chains on rows up to 1024 dims, and k_big_slice (bjx_big.cuh) beyond; initialisation is
// bjx_init_state.  Two routes, chosen from the handle as elliptical slice sampling's are (bjx_ess.cu):
//   rows, [D] scale or [D, D] scale at dim <= 128: the direction is drawn in the warp (the dense one with the small
//     matvec), and the native loop is one persistent launch;
//   big rows (1024 < dim <= 18432), [D] scale: one CTA per chain, the direction in a [C, D] scratch.
#include <math.h>

#include "../../include/bjx.h"
#include "bjx_internal.h"
#include "bjx_big.cuh"
#include "bjx_handle.h"

using namespace bjx;

int bjx_big_slice(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logp_in, float* q_out,
                  float* logp_out, float width, const float* width_dev, const SliceArgs& A);

int bjx_store_scale(bjx_handle_t h, int32_t kind, const float* src, float*& dst, size_t& cap, const char* what) {
  const int D = h->cfg.dim;
  size_t elems;
  if (kind == BJX_METRIC_DIAG) {
    elems = D;
  } else if (kind == BJX_METRIC_DENSE) {
    if (D > 128) return bjx_fail(h, BJX_E_UNSUPPORTED, std::string("a dense ") + what + " is built for dim <= 128");
    elems = (size_t)D * D;
  } else {
    return bjx_fail(h, BJX_E_INVALID, std::string("the ") + what + " has the wrong number of dimensions: expected 1 or 2");
  }
  int rc = bjx_grow(h, dst, cap, elems, sizeof(float));
  if (rc) return rc;
  BJX_CUDA(cudaMemcpyAsync(dst, src, elems * sizeof(float), cudaMemcpyDeviceToDevice, h->stream));
  return 0;
}

extern "C" int bjx_set_slice_direction_scale(bjx_handle_t h, int32_t kind, const float* scale) {
  if (!h || !scale) return bjx_fail(h, BJX_E_INVALID, "null argument");
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  int rc = bjx_store_scale(h, kind, scale, h->slice_scale, h->slice_scale_cap, "slice direction scale");
  if (rc) return rc;
  h->slice_kind = kind;
  return 0;
}

// The route of a call, or the reason it has none: sets big
static int slice_route(bjx_handle_t h, bool& big) {
  if (h->slice_kind < 0)
    return bjx_fail(h, BJX_E_UNSUPPORTED, "slice sampling needs a direction scale: call bjx_set_slice_direction_scale "
                                          "first");
  if (target_route(h) == ROUTE_DENSE)
    return bjx_fail(h, BJX_E_UNSUPPORTED, "slice sampling is not built on the tensor-core dense target path (a dense "
                                          "Gaussian target beyond 128 dims)");
  big = h->sc == SC_BIG;
  if (h->cfg.target.kind == BJX_TARGET_USER) {
    auto* pl = static_cast<bjx_plugin_s*>(h->cfg.target.user_plugin);
    if (big ? !pl->launch_big : !pl->launch)
      return bjx_fail(h, BJX_E_UNSUPPORTED, big ? "slice sampling needs a plug-in built with the big-row kernels "
                                                  "(1024 < dim <= 18432)"
                                                : "slice sampling needs a plug-in built with the row kernels "
                                                  "(dim <= 1024)");
  }
  return 0;
}

static int slice_check(bjx_handle_t h, float width, const float* width_dev, int32_t interval, int32_t max_expansions,
                       int32_t max_shrinkage) {
  if (!width_dev && !(width > 0.f && isfinite(width)))
    return bjx_fail(h, BJX_E_INVALID, "width must be positive and finite");
  if (max_expansions < 0 || max_shrinkage < 0)
    return bjx_fail(h, BJX_E_INVALID, "max_expansions and max_shrinkage must be >= 0");
  if (interval != BJX_SLICE_DOUBLING && interval != BJX_SLICE_STEPPING_OUT)
    return bjx_fail(h, BJX_E_INVALID, "interval must be BJX_SLICE_DOUBLING or BJX_SLICE_STEPPING_OUT");
  return 0;
}

// The arguments every launch shares, with the handle's scratch: the direction [C, D] on the big rows
static int slice_args(bjx_handle_t h, bool big, int32_t interval, int32_t max_expansions, int32_t max_shrinkage,
                      SliceArgs& A) {
  const size_t rows = big ? (size_t)h->cfg.n_chains * h->cfg.dim : 0;
  int rc = bjx_grow(h, h->slice_ws, h->slice_ws_cap, rows, sizeof(float));
  if (rc) return rc;
  A = SliceArgs{};
  A.scale = h->slice_scale;
  A.dir = big ? h->slice_ws : nullptr;
  A.interval = interval;
  A.max_expansions = max_expansions;
  A.max_shrinkage = max_shrinkage;
  return 0;
}

extern "C" int bjx_slice_step(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logp_in,
                              float* q_out, float* logp_out, float width, const float* width_dev, int32_t interval,
                              int32_t max_expansions, int32_t max_shrinkage, const bjx_slice_info* info) {
  const void* ptrs[] = {q_in, q_out};
  int rc = check_ready(h, false, ptrs, 2);
  if (rc) return rc;
  if (!keys || !logp_in || !logp_out) return bjx_fail(h, BJX_E_INVALID, "bad argument");
  if ((rc = slice_check(h, width, width_dev, interval, max_expansions, max_shrinkage))) return rc;
  if ((q_in == q_out) != (logp_in == logp_out))
    return bjx_fail(h, BJX_E_INVALID, "in-place call must alias both of (q, logp)");
  bool big = false;
  if ((rc = slice_route(h, big))) return rc;
  SliceArgs A;
  if ((rc = slice_args(h, big, interval, max_expansions, max_shrinkage, A))) return rc;
  if (info) {
    A.info.is_accepted = info->is_accepted;
    A.info.num_expansions = info->num_expansions;
    A.info.num_shrink = info->num_shrink;
    A.info.bracket_left = info->bracket_left;
    A.info.bracket_right = info->bracket_right;
  }
  if (big) return bjx_big_slice(h, keys, q_in, logp_in, q_out, logp_out, width, width_dev, A);
  LaunchArgs a{};
  a.P = make_params(h, width, width_dev);
  a.keys = keys;
  a.q_in = q_in;
  a.logp_in = logp_in;
  a.q_out = q_out;
  a.logp_out = logp_out;
  a.slice = A;
  return dispatch(h, K_SLICE, true, a);
}

extern "C" int bjx_slice_sample(bjx_handle_t h, const uint32_t* rng_key, float* q, float* logp, int32_t num_steps,
                                float width, const float* width_dev, int32_t interval, int32_t max_expansions,
                                int32_t max_shrinkage, float* history, int32_t thin, int32_t* num_expansions_history,
                                int32_t* num_shrink_history, uint64_t* evaluations) {
  const void* ptrs[] = {q};
  int rc = check_ready(h, false, ptrs, 1);
  if (rc) return rc;
  if (!rng_key || !logp || num_steps < 0 || thin < 1) return bjx_fail(h, BJX_E_INVALID, "bad argument");
  if ((rc = slice_check(h, width, width_dev, interval, max_expansions, max_shrinkage))) return rc;
  bool big = false;
  if ((rc = slice_route(h, big))) return rc;
  if (num_steps == 0) return 0;
  return run_loop(h, rng_key, num_steps, history, thin, [&](const RunLoop& loop) {
    SliceArgs A;
    int rc = slice_args(h, big, interval, max_expansions, max_shrinkage, A);
    if (rc) return rc;
    A.loop = loop;
    A.expansions_history = num_expansions_history;
    A.shrink_history = num_shrink_history;
    A.evaluations = reinterpret_cast<unsigned long long*>(evaluations);
    if (big) return bjx_big_slice(h, nullptr, q, logp, q, logp, width, width_dev, A);
    LaunchArgs a{};
    a.P = make_params(h, width, width_dev);
    a.q_out = q;
    a.logp_out = logp;
    a.slice = A;
    return dispatch(h, K_SLICE_CHAINS, true, a);
  });
}
