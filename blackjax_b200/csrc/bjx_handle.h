// The opaque handle behind include/bjx.h (internal).
#pragma once
#include <string>

#include "../../include/bjx.h"
#include "bjx_internal.h"
#include "bjx_kernels.cuh"

namespace bjx {
struct LaunchArgs;
struct BigLaunchArgs;
}
// A loaded target plug-in (bjx_plugin_load): the warp-kernel launcher (rows up to 1024 dims) and / or the big-row launcher
struct bjx_plugin_s {
  void* dl;
  int (*launch)(int kernel_id, int sc, int dm, const bjx::LaunchArgs* a);
  int (*launch_big)(int kernel_id, const bjx::BigLaunchArgs* a);
};

struct bjx_handle_s {
  bjx_config cfg{};
  cudaStream_t stream = nullptr;
  int sc = 0;                    // SizeClass
  int metric_kind = -1;          // -1 until set
  bool metric_small_dense = false;
  const float* imm = nullptr;    // caller-owned
  float* msqrt = nullptr;        // owned
  size_t msqrt_elems = 0;
  float* chol = nullptr;         // owned: L = chol(M^-1) [D,D] of a dense metric (M^-1/2; Barker's proposal)
  size_t chol_elems = 0;
  // NUTS workspace (owned, lazily allocated)
  bjx::NutsWs ws{};
  void* ws_block = nullptr;
  int ws_depth = 0;
  int* h_flag = nullptr;         // pinned
  int64_t last_leaf_launches = 0, last_depth = 0;
  // large-D dense path (bjx_dense.cu): working rows p, v, q, g [C,D] + GEMM workspace
  float* dense_block = nullptr;
  size_t dense_bytes = 0;
  void* gemm_ws = nullptr;
  size_t gemm_ws_bytes = 0;
  uint16_t* dense_mat_s[4] = {};       // fp16-split copies of M^-1, L^-T, target precision, prior chol(cov) ([D, 3D] each)
  const float* dense_mat_src[4] = {};  // the float32 matrices they were built from
  unsigned dense_mat_ver[4] = {};
  unsigned dense_version = 1;    // bumped by bjx_set_metric / bjx_set_target (contents may change behind the same pointer)
  size_t dense_bytes_built = 0;
  float* lr_block = nullptr;     // low-rank metric (owned): U [D,k] | sigma [D] | 1/sigma [D] | lambda-1 [k] | 1/sqrt(lambda)-1 [k]
  int lr_k = 0;
  void* dn_block = nullptr;      // NUTS on the dense path (bjx_dense_nuts.cuh): compact rows, checkpoint velocities
  size_t dn_bytes = 0;
  float* pool_scratch = nullptr; // scratch of bjx_pooled_stats_dense (slice partials of the D x D co-moment)
  size_t pool_scratch_bytes = 0;
  int ncoef = 3;                 // integrator coefficient table (integrators.py:321-369); {0.5, 1, 0.5} = velocity Verlet
  float coef[11] = {0.5f, 1.0f, 0.5f};
  bool general_integrator = false;
  int key_shared = 0;                  // see bjx_set_key_mode
  const int32_t* steps_dev = nullptr;  // see bjx_set_integration_steps
  const float* steps_avg = nullptr;    // see bjx_set_integration_steps_avg
  const float* ghmc_noise = nullptr;   // see bjx_set_ghmc_noise
  uint32_t chain_offset = 0;
  uint32_t* sample_keys = nullptr;     // [num_steps, 2] step keys of the run loops (bjx_hmc_sample, ...)
  size_t sample_keys_cap = 0;
  int* chain_queue = nullptr;          // the persistent run loops' chain queue (RunLoop::queue), one int
  float* gist_ws = nullptr;            // GIST scratch (bjx_gist.cu): 4 rows [C,D]
  size_t gist_ws_cap = 0;
  // elliptical slice prior (bjx_ess.cu), apart from the metric: kind -1 until set; mean [D] | sqrt(cov) [D] or
  // chol(cov) [D, D]
  int ess_kind = -1;
  float* ess_prior = nullptr;
  size_t ess_prior_cap = 0;
  float* ess_ws = nullptr;             // nu [C, D] of the big rows
  size_t ess_ws_cap = 0;
  // slice sampling's direction scale (bjx_slice.cu): kind -1 until set; [D] or [D, D]
  int slice_kind = -1;
  float* slice_scale = nullptr;
  size_t slice_scale_cap = 0;
  float* slice_ws = nullptr;           // the direction [C, D] of the big rows
  size_t slice_ws_cap = 0;
  // random-walk Metropolis's Gaussian proposal (bjx_rw.cu): kind -1 until set; sigma [D] or [D, D]; mean [D] and
  // 1 / sigma [D] (a [D] sigma)
  int rw_kind = -1;
  int rw_sigma_kind = -1;
  float* rw_sigma = nullptr;
  size_t rw_sigma_cap = 0;
  float* rw_mean = nullptr;      // mean [D] | 1 / sigma [D]
  size_t rw_mean_cap = 0;
  std::string err;
};

int bjx_fail(bjx_handle_t h, int code, const std::string& msg);
int bjx_ensure_nuts_ws(bjx_handle_t h);  // the NUTS workspace of bjx_api.cu (shared with the dense path)
int bjx_cuda_fail(bjx_handle_t h, cudaError_t e, const char* where);
// The [D] (kind BJX_METRIC_DIAG) or [D, D] (BJX_METRIC_DENSE, dim <= 128) float32 device array src copied into the
// handle's grow-only buffer dst on its stream (bjx_slice.cu): slice sampling's direction scale, random-walk Metropolis's
// sigma.  A refusal names the array `what`.
int bjx_store_scale(bjx_handle_t h, int32_t kind, const float* src, float*& dst, size_t& cap, const char* what);

// Grow-only device buffer: *buf holds at least `need` units (elements or bytes, as *cap counts them) afterwards.
template <class T>
int bjx_grow(bjx_handle_t h, T*& buf, size_t& cap, size_t need, size_t unit_bytes) {
  if (need <= cap) return 0;
  if (buf) {
    cudaError_t e = cudaFree(buf);
    buf = nullptr;
    cap = 0;
    if (e != cudaSuccess) return bjx_cuda_fail(h, e, "cudaFree");
  }
  cudaError_t e = cudaMalloc((void**)&buf, need * unit_bytes);
  if (e != cudaSuccess) return bjx_cuda_fail(h, e, "cudaMalloc");
  cap = need;
  return 0;
}

// For its lifetime every chain's key derives from one step key (bjx_set_key_mode 1); the caller's mode comes back after.
struct SharedStepKeys {
  bjx_handle_t h;
  int saved;
  explicit SharedStepKeys(bjx_handle_t h_) : h(h_), saved(h_->key_shared) { h->key_shared = 1; }
  ~SharedStepKeys() { h->key_shared = saved; }
};

inline unsigned blocks_for(long long n, int per_block) { return (unsigned)((n + per_block - 1) / per_block); }

// Stream-ordered device scratch of one call, released on the stream when it goes out of scope.
struct StreamScratch {
  bjx_handle_t h;
  void* ptr = nullptr;
  explicit StreamScratch(bjx_handle_t h_) : h(h_) {}
  ~StreamScratch() {
    if (ptr) cudaFreeAsync(ptr, h->stream);
  }
};

// Chains per slice of the tuners' ESS stage: the most whose position history [n, slice, D] fits max_history_bytes, at least
// one and at most C.
inline long long history_slice_chains(long long max_history_bytes, int n, int D, int C) {
  long long cs = max_history_bytes / ((long long)n * D * (long long)sizeof(float));
  return cs < 1 ? 1 : (cs > C ? C : cs);
}

// Error idiom of every entry point: a failing CUDA call or kernel launch returns its cudaError_t, message in h->err.
#define BJX_CUDA(call)                                            \
  do {                                                            \
    cudaError_t e_ = (call);                                      \
    if (e_ != cudaSuccess) return bjx_cuda_fail(h, e_, #call);    \
  } while (0)
#define BJX_CHECK_LAUNCH(where)                                   \
  do {                                                            \
    cudaError_t e_ = cudaGetLastError();                          \
    if (e_ != cudaSuccess) return bjx_cuda_fail(h, e_, where);    \
  } while (0)

// A native run loop: the step keys split(rng_key, num_steps) into h->sample_keys, then run(loop) with every chain's key
// derived from the step key (SharedStepKeys).
template <class Run>
int run_loop(bjx_handle_t h, const uint32_t* rng_key, int num_steps, float* history, int thin, Run run) {
  int rc = split_step_keys(h, rng_key, num_steps);
  if (rc) return rc;
  SharedStepKeys shared(h);
  return run(bjx::RunLoop{h->sample_keys, num_steps, history, thin, h->chain_queue});
}

// The run loop of one transition per step enqueued from the host: step(t, step key t) for every t, each followed by the
// copy of the positions q into their history row; nothing waits for the device.
template <class Step>
int run_steps(bjx_handle_t h, const uint32_t* rng_key, int num_steps, float* history, int thin, const float* q, Step step) {
  return run_loop(h, rng_key, num_steps, history, thin, [&](const bjx::RunLoop& loop) {
    const size_t row = (size_t)h->cfg.n_chains * h->cfg.dim;
    int rc = 0;
    for (int t = 0; t < num_steps && rc == 0; ++t) {
      rc = step(t, loop.step_keys + 2 * (size_t)t);
      if (rc == 0 && BJX_KEEPS_HISTORY(loop, t))
        BJX_CUDA(cudaMemcpyAsync(BJX_HISTORY_ROW(loop, t, 1, 0, row), q, row * sizeof(float), cudaMemcpyDeviceToDevice,
                                 h->stream));
    }
    return rc;
  });
}

// The tuners' ESS stage, one slice of chains [c0, c0 + n) at a time: n_steps calls of step(c0, n, t), each followed by a
// copy of the slice's positions q into history row t; then the per-chain ESS of the slice into ess [n, D] and
// finish(c0, n).  history holds [n_steps, cs, D] floats, ess [cs, D].
template <class Step, class Finish>
int run_ess_slices(bjx_handle_t h, long long cs, int n_steps, const float* q, float* history, float* ess, Step step,
                   Finish finish) {
  const int C = h->cfg.n_chains, D = h->cfg.dim;
  for (long long c0 = 0; c0 < C; c0 += cs) {
    const int n = (int)((C - c0) < cs ? (C - c0) : cs);
    const size_t row = (size_t)c0 * D;
    for (int t = 0; t < n_steps; ++t) {
      int rc = step(c0, n, t);
      if (rc) return rc;
      BJX_CUDA(cudaMemcpyAsync(history + (size_t)t * n * D, q + row, sizeof(float) * n * D, cudaMemcpyDeviceToDevice,
                               h->stream));
    }
    bjx::launch_ess_per_chain(n_steps, n, D, history, ess, nullptr, h->stream);
    BJX_CHECK_LAUNCH("k_ess_chain");
    int rc = finish(c0, n);
    if (rc) return rc;
  }
  return 0;
}
