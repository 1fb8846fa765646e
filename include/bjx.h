/*
 * bjx.h -- C ABI of the H100-native HMC/NUTS hot path (libbjx.so).
 *
 * Drop-in boundary for BlackJAX's `blackjax.hmc` / `blackjax.nuts` / `window_adaptation`
 * path (reference: blackjax-devs/blackjax @ 63912a4).  The reference has no FFI of its own
 * (it is pure Python on JAX), so every entry point below cites the reference *function* it
 * replaces; `INTEGRATION.md` shows the ctypes binding a maintainer would add.
 *
 * Conventions
 *  - All array pointers are DEVICE pointers owned by the caller unless marked "host".
 *  - State arrays are row-major float32 [n_chains, dim] (chain-major, dimension contiguous);
 *    per-chain scalars are [n_chains]; PRNG keys are uint32 [n_chains, 2] (raw threefry keys,
 *    i.e. jax.random.key_data layout).
 *  - Every call is asynchronous and ordered on the handle's stream (bjx_nuts_step included: the tree doubling is
 *    driven from host C++ as launches whose row counts stay on the device); the only calls that wait for the
 *    device are bjx_synchronize, bjx_destroy, bjx_nuts_last_stats and -- once per tree doubling -- bjx_nuts_step on the
 *    tensor-core dense path (dense metric / dense target with dim > 128: the products are sized from the row count).
 *  - Return value: 0 ok; <0 invalid argument / unsupported configuration (BJX_E_*);
 *    >0 a cudaError_t.  bjx_last_error(handle) returns the text.  No exceptions or
 *    callbacks cross this ABI.  A handle is not thread-safe; distinct handles are independent.
 *  - There is NO CPU fallback: every entry point fails with a CUDA error if no device exists.
 */
#ifndef BJX_H_
#define BJX_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BJX_VERSION 100

/* error codes (negative) */
#define BJX_OK 0
#define BJX_E_INVALID (-1)     /* bad argument / shape */
#define BJX_E_UNSUPPORTED (-2) /* configuration not built (e.g. dim % 4 != 0 with dim > 128) */
#define BJX_E_STATE (-3)       /* call order (e.g. metric not set) */

/* log-density targets with a fused analytic value_and_grad (replaces jax.value_and_grad of the
 * user callable: blackjax/mcmc/hmc.py:91, integrators.py:189,204). */
enum bjx_target_kind {
  BJX_TARGET_DIAG_GAUSSIAN = 0,  /* -1/2 sum ((x-mean)/s)^2 + offset   tests/fixtures.py:60-78   */
  BJX_TARGET_FUNNEL = 1,         /* Neal's funnel                       tests/fixtures.py:81-98   */
  BJX_TARGET_DENSE_GAUSSIAN = 2, /* -1/2 x^T P x + offset               tests/mcmc/test_mclmc_lrd.py:86-88 */
  BJX_TARGET_BANANA = 3,         /* -(1-x0)^2 - 1.5 (x1-x0^2)^2, dim=2  tests/mcmc/test_trajectory.py:79-80 */
  BJX_TARGET_HIER_LOGIT = 4,     /* hierarchical logistic regression (BASELINE config 5; builder-defined, see
                                    DESIGN.md): x = [mu, log tau, beta0, beta1, alpha_0..alpha_{G-1}], dim = 4 + G */
  BJX_TARGET_USER = 5            /* user-defined value_and_grad compiled into a plug-in (bjx_plugin_load; dim <= 1024):
                                    the slot of the arbitrary `logdensity_fn` callable of hmc.py:91 / nuts.py:133 */
};

/* inverse-mass-matrix layouts (metrics.py:701-729: 1-D => diagonal, 2-D => dense) */
enum bjx_metric_kind {
  BJX_METRIC_DIAG = 0,          /* imm [dim]                                    */
  BJX_METRIC_DENSE = 1,         /* imm [dim, dim] symmetric positive definite   */
  BJX_METRIC_DIAG_PER_CHAIN = 2, /* imm [n_chains, dim] (vmapped window adaptation) */
  BJX_METRIC_LOW_RANK = 3,       /* bjx_set_metric_low_rank */
  BJX_METRIC_DENSE_PER_CHAIN = 4 /* imm [n_chains, dim, dim], dim <= 64 (vmapped dense window adaptation) */
};

typedef struct {
  int32_t kind;           /* bjx_target_kind */
  int32_t dim;
  const float* inv_var;   /* DIAG_GAUSSIAN: [dim] 1/s^2 (device)           */
  const float* mean;      /* DIAG_GAUSSIAN: [dim] or NULL (device)         */
  const float* precision; /* DENSE_GAUSSIAN: [dim, dim] symmetric (device) */
  float logp_offset;      /* constant added to every log-density           */
  const float* data_x;    /* HIER_LOGIT: covariates [G, 8, 2] (device)     */
  const uint8_t* data_y;  /* HIER_LOGIT: outcomes, bit k of byte g = y_gk  */
  int32_t n_groups;       /* HIER_LOGIT: G (dim = 4 + G)                   */
  int32_t n_user_params;  /* USER: floats in user_params                   */
  const float* user_params; /* USER: parameter block (device) or NULL      */
  void* user_plugin;      /* USER: plug-in from bjx_plugin_load            */
} bjx_target_desc;

typedef struct {
  int32_t device;              /* CUDA ordinal */
  int32_t n_chains;            /* chains held by THIS process/GPU */
  int32_t dim;
  int32_t max_tree_depth;      /* NUTS checkpoint capacity (max_num_doublings upper bound), >= 1 */
  float divergence_threshold;  /* default 1000 (hmc.py:120, trajectory.py:325) */
  void* stream;                /* cudaStream_t to order all work on (NULL = legacy default stream) */
  bjx_target_desc target;
} bjx_config;

/* Optional per-transition outputs (NULL => not written).  Mirrors HMCInfo (hmc.py:52-87) and
 * NUTSInfo (nuts.py:36-74); D-sized fields only on request. */
typedef struct {
  float* acceptance_rate;          /* [C]                                              */
  uint8_t* is_accepted;            /* [C]   HMC only                                   */
  uint8_t* is_divergent;           /* [C]                                              */
  uint8_t* is_turning;             /* [C]   NUTS only                                  */
  float* energy;                   /* [C]   energy of the proposal                     */
  int32_t* num_integration_steps;  /* [C]                                              */
  int32_t* num_trajectory_expansions; /* [C] NUTS only                                 */
  float* momentum;                 /* [C,D] momentum drawn at the start of the transition */
  float* proposal_position;        /* [C,D] HMC: end state (before accept/reject)      */
  float* proposal_momentum;        /* [C,D] HMC: flipped end momentum                  */
  float* left_position;            /* [C,D] NUTS trajectory_leftmost_state.position    */
  float* left_momentum;            /* [C,D]                                            */
  float* right_position;           /* [C,D] NUTS trajectory_rightmost_state.position   */
  float* right_momentum;           /* [C,D]                                            */
} bjx_info;

typedef struct bjx_handle_s* bjx_handle_t;

/* ---- lifecycle ------------------------------------------------------------------------------ */
int bjx_version(void);
int bjx_create(const bjx_config* cfg, bjx_handle_t* out);
int bjx_destroy(bjx_handle_t h);
const char* bjx_last_error(bjx_handle_t h); /* h may be NULL: last global error */
int bjx_set_target(bjx_handle_t h, const bjx_target_desc* target);
/* User-defined targets.  BlackJAX takes any callable and differentiates it (`jax.value_and_grad(logdensity_fn)`,
 * mcmc/hmc.py:91, integrators.py:189); here the plug-in point is the fused value_and_grad device function
 * (`bjx_user::Model<R>::value_and_grad`, contract in include/bjx_user_target.h).  A plug-in is a small shared library built from
 * blackjax_b200/csrc/bjx_plugin.cu + the user's source (nvcc; blackjax_b200/plugin.py does it from Python) holding every
 * transition kernel of the path instantiated around that function.  bjx_plugin_load opens it (host path), checks that it
 * was built against this library's kernel ABI (bjx_plugin_abi) and returns the pointer to put into
 * bjx_target_desc.user_plugin with kind = BJX_TARGET_USER.  Plug-ins stay loaded for the life of the process. */
int bjx_plugin_load(const char* path, void** plugin_out);
int bjx_plugin_abi(void);
/* Palindromic two-stage integrator (integrators.py:62-152): host array of n coefficients, n odd in 3..11.
 * {0.5, 1, 0.5} = velocity_verlet (default, :321-322); mclachlan :335-340, yoshida :351-357, omelyan :363-369. */
int bjx_set_integrator(bjx_handle_t h, const float* coefficients, int32_t n);
/* Key source for bjx_sample_momentum / bjx_hmc_step / bjx_mhmc_step / bjx_nuts_step: shared_step_key = 0 (default):
 * `keys` is uint32 [n_chains, 2], one rng_key per chain.  shared_step_key = 1: `keys` is ONE key uint32 [2] and
 * chain c uses jax.random.split(key, n_global)[chain_offset + c] (= fold_in(key, chain_offset + c)), derived inside the
 * kernel -- the reference's step-major schedule (docs/examples/howto_sample_multiple_chains.md:116-129), independent
 * of how the chains are sharded over GPUs (chain_offset = first global chain of this handle). */
int bjx_set_key_mode(bjx_handle_t h, int32_t shared_step_key, uint32_t chain_offset);
/* Dynamic HMC (blackjax/mcmc/dynamic_hmc.py:62-130): every chain integrates its own number of steps.  steps_dev: int32
 * [n_chains] device array read by the following bjx_hmc_step / bjx_mhmc_step calls (their scalar L is then ignored);
 * NULL restores the scalar.  The caller keeps the array alive until those calls have run.  dim <= 1024 only. */
int bjx_set_integration_steps(bjx_handle_t h, const int32_t* steps_dev);
/* Adjusted MCLMC with one average trajectory length per chain (e.g. the tuner's L / step_size): float32 [n_chains] device
 * array read by the following bjx_adjusted_mclmc_step / bjx_adjusted_mclmc_sample calls.  BJX_AMCLMC_STEPS_FIXED then runs
 * ceil(avg[c]) steps (in place of num_integration_steps and bjx_set_integration_steps), BJX_AMCLMC_STEPS_UNIFORM scales by
 * rescale(avg[c]) in float32 (in place of steps_scale); RANDINT ignores it.  NULL restores the scalar arguments.  The caller
 * keeps the array alive until those calls have run. */
int bjx_set_integration_steps_avg(bjx_handle_t h, const float* avg_dev);
/* Generalized HMC slice noise (mcmc/ghmc.py:90,172 `noise_fn(key_noise)`, key_noise = split(rng_key)[1]): per-chain values
 * float32 [C] (device) for the following bjx_ghmc_step calls, evaluated by the caller; NULL = the default noise_fn (0). */
int bjx_set_ghmc_noise(bjx_handle_t h, const float* noise_dev);
int bjx_synchronize(bjx_handle_t h);

/* metrics.default_metric / gaussian_euclidean (metrics.py:180-218,221-346): precomputes
 * mass_matrix_sqrt = 1/sqrt(M^-1) (diag) or L^-T with L = chol(M^-1) (dense), metrics.py:701-729.
 * The dense factorisation runs on the host in float64 and synchronises the stream. */
int bjx_set_metric(bjx_handle_t h, int32_t metric_kind, const float* inverse_mass_matrix);
/* metrics.gaussian_euclidean_low_rank(sigma, U, lam) (metrics.py:349-467): M^-1 = diag(sigma) (I + U (Lambda - I) U^T) diag(sigma),
 * sigma [dim] > 0, U [dim, rank] row-major with orthonormal columns, lam [rank] > 0 (device arrays, copied).  Momentum
 * draw, kinetic energy, velocity and the U-turn test all cost O(dim * rank).  rank <= 16, dim <= 512 (warp kernels: HMC,
 * multinomial HMC, NUTS). */
int bjx_set_metric_low_rank(bjx_handle_t h, const float* sigma, const float* U, const float* lam, int32_t rank);
/* device pointer to mass_matrix_sqrt as precomputed by bjx_set_metric (for tests) */
int bjx_get_mass_matrix_sqrt(bjx_handle_t h, const float** out);

/* ---- building blocks (KAT-able; each maps to one reference function) -------------------------- */
/* hmc.init (hmc.py:90-92): logp, grad = value_and_grad(logdensity)(q) */
int bjx_init_state(bjx_handle_t h, const float* q, float* logp_out, float* grad_out);
/* metric.sample_momentum (metrics.py:260-261 -> util.py:66-91): p = mass_matrix_sqrt (.) normal(key,(D,)) */
int bjx_sample_momentum(bjx_handle_t h, const uint32_t* keys, float* p_out);
/* static_integration (trajectory.py:136-167) of velocity_verlet (integrators.py:62-152,321-322):
 * n_steps leapfrogs in place.  step_size_dev ([C], signed) overrides step_size when non-NULL. */
int bjx_leapfrog(bjx_handle_t h, float* q, float* p, float* logp, float* grad, float step_size,
                 const float* step_size_dev, int32_t n_steps);
/* linear_map(inverse_mass_matrix, p) (blackjax/util.py:23-61; the kinetic-energy gradient of
 * integrators.py:242): v = M^-1 p for every chain.  Dense metric with dim > 128: one tensor-core GEMM. */
int bjx_metric_velocity(bjx_handle_t h, const float* p, float* v_out);
/* hmc_energy (trajectory.py:730-750): -logp + 1/2 p^T M^-1 p */
int bjx_energy(bjx_handle_t h, const float* p, const float* logp, float* energy_out);
/* metrics.is_turning (metrics.py:272-304) on explicit momenta (for the U-turn truth table) */
int bjx_is_turning(bjx_handle_t h, const float* p_left, const float* p_right, const float* p_sum,
                   uint8_t* out);

/* ---- transitions ------------------------------------------------------------------------------ */
/* hmc.build_kernel(...).kernel (hmc.py:279-312).  (q,logp,grad)_in -> (q,logp,grad)_out; out may
 * alias in (in-place).  keys: one rng_key per chain. */
int bjx_hmc_step(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logp_in,
                 const float* grad_in, float* q_out, float* logp_out, float* grad_out,
                 float step_size, const float* step_size_dev, int32_t num_integration_steps,
                 const bjx_info* info);
/* Multinomial HMC: hmc.build_kernel(build_proposal=multinomial_hmc_proposal) = blackjax.mhmc (hmc.py:181-248,
 * trajectory.py:170-232, blackjax/__init__.py:145-151).  Same arguments as bjx_hmc_step; is_accepted is always 1,
 * acceptance_rate = exp(sum_log_p_accept) / L, proposal_* = the selected trajectory state. */
int bjx_mhmc_step(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logp_in,
                  const float* grad_in, float* q_out, float* logp_out, float* grad_out,
                  float step_size, const float* step_size_dev, int32_t num_integration_steps,
                  const bjx_info* info);
/* Generalized HMC: ghmc.build_kernel().kernel (blackjax/mcmc/ghmc.py:118-189; update_momentum :192-213;
 * nonreversible_slice_sampling blackjax/mcmc/proposal.py:243-264), in place on the persistent state
 * (q [C,D], p [C,D], logp [C], grad [C,D], slice [C]); noise_fn is the reference default (0).
 * step_size_dev / alpha_dev / delta_dev (optional) are indexed by chain / chains_per_group; imm_rows + msqrt_rows
 * (optional, [C / chains_per_group, D]: inverse mass = momentum_inverse_scale^2, ghmc.py:83-84, and 1/sqrt of it)
 * override the handle's diagonal metric row-wise -- MEADS' per-fold parameters (meads_adaptation.py:587-606).
 * Chains in [skip_begin, skip_end) are computed but keep their state (the frozen fold, :639-650). */
int bjx_ghmc_step(bjx_handle_t h, const uint32_t* keys, float* q, float* p, float* logp, float* grad, float* slice,
                  float step_size, const float* step_size_dev, float alpha, const float* alpha_dev, float delta,
                  const float* delta_dev, const float* imm_rows, const float* msqrt_rows, int32_t chains_per_group,
                  int32_t skip_begin, int32_t skip_end, const bjx_info* info);
/* MEADS fold statistics and parameters (blackjax/adaptation/meads_adaptation.py:507-585, maximum_eigenvalue :787-817)
 * from the positions and gradients of all chains, folds = contiguous blocks of C / num_folds chains, t = the
 * adaptation iteration.  state float32 [bjx_meads_state_floats] = step_size[K] | alpha[K] | delta[K] | sigma[K,D] |
 * imm[K,D] | msqrt[K,D], already rolled by one fold (:560-563), i.e. the arrays bjx_ghmc_step takes.
 * num_folds = 1 gives base.compute_parameters (:97-152) of all chains. */
size_t bjx_meads_state_floats(int32_t num_folds, int32_t dim);
size_t bjx_meads_scratch_floats(int32_t n_chains, int32_t dim, int32_t num_folds);
int bjx_meads_update(bjx_handle_t h, const float* q, const float* grad, int32_t num_folds, int32_t t,
                     float step_size_multiplier, float damping_slowdown, float* state, float* scratch);
/* MEADS-LRD (meads_adaptation.py:459-784 with low_rank_rank = k): ONE low-rank metric for all chains per warm-up step.
 * The handle must hold a rank-k low-rank metric (bjx_set_metric_low_rank, installed once with the fallback values);
 * bjx_meads_lrd_update rewrites that metric's block in place on the stream (no allocation, no host round trip).
 * Built for dim <= 512, 1 <= k <= min(16, dim), one GPU; otherwise BJX_E_UNSUPPORTED.
 * lrd_state float32 [bjx_meads_lrd_state_floats], zero-filled before the first step; its first 16 floats are
 *   [0] 1 if this step's metric came from the accumulator   [1] eigensolver iterations of the last solve
 *   [2] its largest residual ||A u - mu u|| / max|mu|       [3] 1 once any solve stopped at the iteration cap (sticky)
 *   [4] sum and [5] maximum of the iterations over solves   [6] number of solves   [7] 1 once a Ritz basis is stored
 * followed by sigma[D] | U[D,k] | lam[k], the metric of the last step.  scratch: bjx_meads_lrd_scratch_floats.
 * k is read from the handle's low-rank metric on every call: an lrd_state sized for (C, D, k) must only be used
 * with a handle of C chains and D dims holding a rank-k metric (a different rank would address the state wrongly).
 * bjx_meads_lrd_update: with in_window, folds q [C,D] into the windowed covariance accumulator (cgl_update_batch);
 * the metric is the top-k pairs by |lam - 1| of the accumulated correlation matrix when in_window and it holds
 * >= 2 dim samples, else the fallback (std of q over all chains, pooled from the per-fold mean and std, so equal
 * to a direct std up to float32 rounding; eye(dim, k), ones(k)); lam floored at 1e-6.  state
 * as in bjx_meads_update: the step sizes are those of bjx_meads_update, alpha / delta come from the fold-centred
 * positions under the low-rank transform (x + ((x U)(lam^-1/2 - 1)) U^T) / sigma (:599-634).  Run bjx_ghmc_step with
 * the state's step_size / alpha / delta rows and imm_rows = msqrt_rows = NULL.
 * bjx_meads_lrd_metric: the final metric (:746-771) -- the accumulator if it holds >= 2 dim samples, else the
 * fallback on final_q -- into sigma_out [D], U_out [D,k], lam_out [k] (device). */
size_t bjx_meads_lrd_state_floats(int32_t n_chains, int32_t dim, int32_t rank);
size_t bjx_meads_lrd_scratch_floats(int32_t n_chains, int32_t dim, int32_t num_folds);
int bjx_meads_lrd_update(bjx_handle_t h, const float* q, const float* grad, int32_t num_folds, int32_t t, int32_t in_window,
                         float step_size_multiplier, float damping_slowdown, float* state, float* lrd_state, float* scratch);
int bjx_meads_lrd_metric(bjx_handle_t h, float* lrd_state, const float* final_q, float* sigma_out, float* U_out,
                         float* lam_out);
/* maximum_eigenvalue (meads_adaptation.py:787-817) of one float32 [n, d] device matrix; out: ONE device float */
size_t bjx_maximum_eigenvalue_scratch_floats(int64_t n, int32_t d);
int bjx_maximum_eigenvalue(bjx_handle_t h, const float* x, int64_t n, int32_t d, float* out, float* scratch);
/* jax.random.permutation(key', n) with key' = fold_in(key, fold_index) (fold_index < 0: key itself): the sort-based
 * shuffle of jax/_src/random.py.  perm_out int32 [n]; scratch: bjx_permutation_scratch_bytes(n) bytes. */
size_t bjx_permutation_scratch_bytes(int64_t n);
int bjx_permutation(bjx_handle_t h, const uint32_t* key, int64_t fold_index, int64_t n, int32_t* perm_out, void* scratch);
/* dst[r, :] = src[perm[r], :] for float32 [rows, width] (the shuffle of meads_adaptation.py:675-683); out of place */
int bjx_gather_rows(bjx_handle_t h, const int32_t* perm, const float* src, float* dst, int64_t rows, int32_t width);
/* blackjax.util.run_inference_algorithm (util.py:150-213) for HMC (multinomial = 0) / multinomial HMC (1), run
 * natively: step keys = jax.random.split(rng_key, num_steps) (util.py:203), num_steps in-place transitions enqueued back
 * to back without host synchronisation; chain c of step t uses split(step_key_t, n_global)[chain_offset + c].
 * rng_key: ONE key uint32 [2] (device).  history (optional): float32 [num_steps / thin, C, D], the positions after every
 * thin-th transition; acceptance_history (optional): float32 [num_steps, C]. */
int bjx_hmc_sample(bjx_handle_t h, const uint32_t* rng_key, float* q, float* logp, float* grad, float step_size,
                   const float* step_size_dev, int32_t num_integration_steps, int32_t num_steps, int32_t multinomial,
                   float* history, int32_t thin, float* acceptance_history);
/* nuts.build_kernel(...).kernel (nuts.py:113-145) with iterative_nuts_proposal (nuts.py:223-321).
 * Tree doubling is driven from the host: one launch per doubling over the chains still expanding; each
 * warp integrates its chain's whole sub-tree (up to 2^d leapfrog leaves) inside the launch.
 * Dense metric / dense Gaussian target with 128 < dim <= 1024: the chains of a doubling advance through its leaves in lock
 * step, compacted, on the tensor-core products (three per leaf: half-step velocity, gradient, full-step velocity for the
 * energy and the U-turn tests, metrics.py:263-304); same keys and decisions.
 * momentum_override/key_integrator_override (both or neither, for KATs): skip the key split and
 * the momentum draw and use the given momentum [C,D] and integrator keys [C,2]. */
int bjx_nuts_step(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logp_in,
                  const float* grad_in, float* q_out, float* logp_out, float* grad_out,
                  float step_size, const float* step_size_dev, int32_t max_num_doublings,
                  const bjx_info* info, const float* momentum_override,
                  const uint32_t* key_integrator_override);
/* blackjax.util.run_inference_algorithm (util.py:150-213) for NUTS, run natively like bjx_hmc_sample: step keys =
 * split(rng_key, num_steps), transitions in place, no host synchronisation.  With num_steps >= 4 the chains run DECOUPLED:
 * one persistent launch whose warps take whole chains through all transitions (chains never interact and transition t
 * of chain c needs only step key t), bit-identical to num_steps calls of bjx_nuts_step.  history (optional) float32
 * [num_steps / thin, C, D]; acceptance_history (optional) float32 [num_steps, C]; num_integration_steps_history (optional)
 * int32 [num_steps, C]. */
int bjx_nuts_sample(bjx_handle_t h, const uint32_t* rng_key, float* q, float* logp, float* grad, float step_size,
                    const float* step_size_dev, int32_t max_num_doublings, int32_t num_steps, float* history, int32_t thin,
                    float* acceptance_history, int32_t* num_integration_steps_history);
/* doubling launches and the deepest tree of the last bjx_nuts_step (host ints; reading the depth synchronises the stream) */
int bjx_nuts_last_stats(bjx_handle_t h, int64_t* doubling_launches, int64_t* depth_reached);

/* ---- MCLMC: the microcanonical Langevin sampler (blackjax/mcmc/mclmc.py) -------------------------------------------
 * State (q [C,D], p [C,D], logp [C], grad [C,D]); p is the unit-norm momentum of the whitened frame.  The metric must be
 * BJX_METRIC_DIAG or BJX_METRIC_DIAG_PER_CHAIN (the preconditioner is sqrt(M^-1), integrators.py:437-439); the integrator is
 * the handle's coefficient table run as the isokinetic integrator (isokinetic_mclachlan = the mclachlan table,
 * integrators.py:533-539).  Built for 2 <= dim <= 1024 (dense Gaussian target: dim <= 128); everything else returns
 * BJX_E_UNSUPPORTED.  Keys follow bjx_set_key_mode. */
typedef struct {
  float* kinetic_change; /* [C] MCLMCInfo.kinetic_change (0 on a reverted transition) */
  float* energy_change;  /* [C] kinetic_change - logp_new + logp_old (0 on a reverted transition) */
  uint8_t* nonans;       /* [C] 1 when q, p and logp came out finite */
} bjx_mclmc_info;
/* mclmc.init (mclmc.py:55-66): logp, grad = value_and_grad(q); p = generate_unit_vector(key) (util.py:94-113) */
int bjx_mclmc_init(bjx_handle_t h, const uint32_t* keys, const float* q, float* logp_out, float* grad_out, float* p_out);
/* mclmc.build_kernel(...).kernel (mclmc.py:104-143), in place on (q, p, logp, grad).  step_size_dev / L_dev ([C], optional)
 * override step_size / L; L = inf leaves the momentum unrefreshed.  energy_cutoff = sqrt(dim * desired_energy_var_max_ratio *
 * desired_energy_var) (inf by default): a transition with |energy_change| above it, or with a non-finite q, p or logp, keeps
 * (q, logp, grad) and draws a fresh unit momentum (handle_high_energy / handle_nans, mclmc.py:215-281). */
int bjx_mclmc_step(bjx_handle_t h, const uint32_t* keys, float* q, float* p, float* logp, float* grad, float step_size,
                   const float* step_size_dev, float L, const float* L_dev, float energy_cutoff, const bjx_mclmc_info* info);
/* run_inference_algorithm (util.py:150-213) for MCLMC, like bjx_hmc_sample: step keys = split(rng_key, num_steps), chain c
 * of step t uses split(step_key_t, n_global)[chain_offset + c], no host synchronisation.  history (optional) float32
 * [num_steps / thin, C, D]; energy_change_history (optional) float32 [num_steps, C]. */
int bjx_mclmc_sample(bjx_handle_t h, const uint32_t* rng_key, float* q, float* p, float* logp, float* grad, float step_size,
                     const float* step_size_dev, float L, const float* L_dev, float energy_cutoff, int32_t num_steps,
                     float* history, int32_t thin, float* energy_change_history);

/* ---- MCLMC tuning: mclmc_find_L_and_step_size (blackjax/adaptation/mclmc_adaptation.py:42-399) -----------------------
 * Every chain runs the reference's single-chain tuner with its own key, as jax.vmap over chains would, and ends with its own
 * (L, step_size, inverse_mass_matrix).  Supported configurations are those of bjx_mclmc_step (BJX_E_UNSUPPORTED otherwise).
 * The tuner constants are the reference's Python floats: desired_energy_var, trust_in_estimate and num_effective_samples
 * enter as D * desired_energy_var, 6 * trust_in_estimate and (n - 1) / (n + 1), formed in double and rounded to float32. */
/* One tuning step (predictor + step, mclmc_adaptation.py:223-301) in place, for every chain.  keys (per bjx_set_key_mode)
 * give each chain's step key k; (rng_key, nan_key) = split(k), and rng_key drives the transition with L / L_dev and the
 * handle's metric.  A chain whose transition has nonans = 0 or a non-finite energy change keeps its whole previous state
 * (momentum included, or generate_unit_vector(nan_key) when the transition's logdensity is NaN) and sets
 * step_size_max = 0.8 step_size; otherwise it takes nan_to_num of the new state.  step_size, time, x_average and
 * step_size_max ([C] float32, in/out) are the predictor's per-chain scalars; the new step size is
 * (x_average / time)^(-1/6) clipped against step_size_max (0 where equal or NaN, as XLA evaluates the reference's
 * predicate products).  With mask = 1, total [C] and moments [C, 2, D] (in/out; 16-byte aligned) take the streaming
 * average of (x, x^2) with weight success * new step size (incremental_value_update, util.py:287-319); with mask = 0 or
 * moments NULL neither is touched.  success (optional) [C] uint8. */
int bjx_mclmc_tune_step(bjx_handle_t h, const uint32_t* keys, float* q, float* p, float* logp, float* grad, float* step_size,
                        float L, const float* L_dev, float energy_cutoff, float* time, float* x_average, float* step_size_max,
                        float* total, float* moments, int32_t mask, double desired_energy_var, double trust_in_estimate,
                        double num_effective_samples, uint8_t* success);
/* effective_sample_size(history[:, c, None, :]) for every chain: history float32 [num_samples, C, D] (C, D of the handle),
 * ess_out [C, D] single-chain ESS.  Evaluates the autocovariance only up to the lags Geyer's initial positive sequence
 * reads, with the result of evaluating all of them.  lags_evaluated (optional) [C]: the most lags any series of the chain
 * needed, in blocks of 32.  Needs no scratch. */
int bjx_mclmc_ess_per_chain(bjx_handle_t h, const float* history, int32_t num_samples, float* ess_out, int32_t* lags_evaluated);
/* mclmc_find_L_and_step_size, all three stages on the handle's stream with no host synchronisation.  rng_key per
 * bjx_set_key_mode: one key [2] (chain c: split(rng_key, n_global)[chain_offset + c]) or per-chain keys [C, 2].  The host
 * computes the stage lengths: num_steps1 = round(N f1), num_steps2 = round(N f2), readjust_steps = round(num_steps2 / 3),
 * num_steps3 = round(N f3) (Python's round).  step_size [C], L [C] and inverse_mass_matrix [C, D] (a per-chain diagonal
 * metric, used in place of the handle's, which must still be a diagonal kind) are the initial parameters in and the tuned
 * ones out; q, p, logp, grad the state.  Stages 1 and 2 run num_steps1 + num_steps2 tuning steps with the initial L,
 * estimating the moments over the last num_steps2.  If num_steps2 > 1: L = sqrt(sum var), or with
 * diagonal_preconditioning inverse_mass_matrix = var, L = sqrt(D) and readjust_steps more tuning steps (initial L, the new
 * metric).  If num_steps3 >= 2: num_steps3 transitions with the tuned parameters and L = l_factor * step_size *
 * mean(num_steps3 / ESS), run on slices of chains whose position history [num_steps3, slice, D] fits max_history_bytes
 * (at least one chain); the result does not depend on the slice size.  energy_cutoff as in bjx_mclmc_step.
 * divergence_history (optional) uint8 [num_steps1 + num_steps2 (+ readjust_steps when they run), C]: 1 where a tuning
 * step failed (the reference's scan output). */
int bjx_mclmc_find_l_and_step_size(bjx_handle_t h, const uint32_t* rng_key, float* q, float* p, float* logp, float* grad,
                                   float* step_size, float* L, float* inverse_mass_matrix, int32_t num_steps1,
                                   int32_t num_steps2, int32_t readjust_steps, int32_t num_steps3,
                                   int32_t diagonal_preconditioning, float energy_cutoff, double desired_energy_var,
                                   double trust_in_estimate, double num_effective_samples, double l_factor,
                                   int64_t max_history_bytes, uint8_t* divergence_history);

/* ---- Adjusted MCLMC / MAMS: the Metropolis-adjusted microcanonical sampler (blackjax/mcmc/adjusted_mclmc.py,
 * adjusted_mclmc_dynamic.py) ----------------------------------------------------------------------------------------
 * State (q [C,D], logp [C], grad [C,D]) as HMC's; initialise it with bjx_init_state.  One transition draws a unit momentum
 * from split(key)[0], runs num_integration_steps steps of the handle's coefficient table as the isokinetic integrator, each
 * between two partial momentum refreshes with L_proposal = L_proposal_factor * num_integration_steps * step_size (none when
 * L_proposal_factor = inf), and accepts with Metropolis-Hastings; there is no momentum flip.  Per-chain step counts come from
 * bjx_set_integration_steps (adjusted_mclmc_dynamic); 0 steps is allowed and accepts the unchanged state.  bjx_info as HMCInfo:
 * energy = -logp of the proposal, momentum = the drawn unit vector, proposal_momentum = the unflipped end momentum.
 * Same support as MCLMC: diagonal metrics, 2 <= dim <= 1024 (dense Gaussian target: dim <= 128), else BJX_E_UNSUPPORTED.
 * Keys follow bjx_set_key_mode.  A rejected in-place transition writes nothing. */
int bjx_adjusted_mclmc_step(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logp_in,
                            const float* grad_in, float* q_out, float* logp_out, float* grad_out, float step_size,
                            const float* step_size_dev, int32_t num_integration_steps, float L_proposal_factor,
                            const bjx_info* info);
/* Step-count rules of bjx_adjusted_mclmc_sample, evaluated on the device from each chain's random_generator_arg key, which
 * then advances to split(key)[1] (adjusted_mclmc_dynamic.py:58,124):
 *   BJX_AMCLMC_STEPS_FIXED    num_integration_steps for every chain (adjusted_mclmc), random_generator_arg unused;
 *   BJX_AMCLMC_STEPS_RANDINT  jax.random.randint(key, (), 1, 10) (adjusted_mclmc_dynamic.py:55);
 *   BJX_AMCLMC_STEPS_UNIFORM  max(ceil(uniform(key) * steps_scale), min_steps), steps_scale = rescale(avg) in float32
 *                             (adjusted_mclmc_dynamic.py:234-238 with min_steps = 1; the reference's own tests use 0). */
#define BJX_AMCLMC_STEPS_FIXED 0
#define BJX_AMCLMC_STEPS_RANDINT 1
#define BJX_AMCLMC_STEPS_UNIFORM 2
/* run_inference_algorithm (util.py:150-213) for adjusted MCLMC, like bjx_hmc_sample: step keys = split(rng_key, num_steps),
 * no host synchronisation.  random_generator_arg uint32 [C, 2] (rules other than FIXED) is advanced in place.  history
 * (optional) float32 [num_steps / thin, C, D]; acceptance_history (optional) float32 [num_steps, C];
 * steps_history (optional) int32 [num_steps, C]. */
int bjx_adjusted_mclmc_sample(bjx_handle_t h, const uint32_t* rng_key, float* q, float* logp, float* grad, float step_size,
                              const float* step_size_dev, float L_proposal_factor, int32_t steps_rule,
                              int32_t num_integration_steps, float steps_scale, int32_t min_steps,
                              uint32_t* random_generator_arg, int32_t num_steps, float* history, int32_t thin,
                              float* acceptance_history, int32_t* steps_history);
/* The step count int32 [C] of steps_rule for every chain, as the transitions evaluate it, from avg [C] (fixed: ceil(avg),
 * uniform: rescale(avg); randint: unused, may be NULL) and random_generator_arg [C, 2] (unused by the fixed rule, not
 * advanced): max(rule, min_steps). */
int bjx_adjusted_mclmc_num_steps(bjx_handle_t h, int32_t steps_rule, const float* avg, int32_t min_steps,
                                 const uint32_t* random_generator_arg, int32_t* steps_out);

/* ---- GIST: Gibbs self-tuning HMC (blackjax/mcmc/composed: gist_trajectory_length, gist_step_size) --------------------
 * State (q [C,D], logp [C], grad [C,D]) as HMC's; initialise it with bjx_init_state.  One transition draws the momentum
 * (key_momentum = split(key, 3)[0]), draws the tuning parameter given (q, p) (key_tuning = [1]), integrates, re-runs the
 * same choice from the flipped proposal and accepts with uniform(key_accept = [2]) < exp(min(delta + log_ratio, 0)).
 *   BJX_GIST_TRAJECTORY_LENGTH: U = steps until dot(q_n - q_0, p_n) < 0 or max_num_steps; L ~ randint(lo, U + 1) with
 *     lo = max(1, floor(path_fraction * U)) in float32; the log ratio compares the widths of the forward and reverse
 *     intervals, -inf when L is outside the reverse one (is_no_return_rejected).
 *   BJX_GIST_STEP_SIZE: step size step_size * 2^j chosen by the doubling / halving search of at most max_search_steps + 1
 *     trial trajectories of num_integration_steps steps (criterion BJX_GIST_SYMMETRIC or BJX_GIST_ASYMMETRIC); the
 *     transition rejects unless the search from the proposal picks the same j and neither search was exhausted.
 * Built on the warp-per-chain rows (dim <= 1024) with every row metric, target and integrator table there; dim > 1024 and
 * the tensor-core dense path (a dense metric or dense Gaussian target beyond 128 dims) return BJX_E_UNSUPPORTED.  The
 * handle keeps a scratch of 4 rows [C,D] (the initial momentum and the proposal) instead of the rollout, which is
 * re-integrated: a transition costs about U + L + N gradient evaluations (trajectory length) or the trial steps of both
 * searches plus num_integration_steps (step size). */
#define BJX_GIST_TRAJECTORY_LENGTH 0
#define BJX_GIST_STEP_SIZE 1
#define BJX_GIST_SYMMETRIC 0
#define BJX_GIST_ASYMMETRIC 1
typedef struct {
  int32_t instance;              /* BJX_GIST_TRAJECTORY_LENGTH or BJX_GIST_STEP_SIZE */
  float path_fraction;           /* trajectory length: psi in [0, 1] (0.5) */
  int32_t max_num_steps;         /* trajectory length: cap on each rollout, >= 1 (1024) */
  int32_t num_integration_steps; /* step size: steps per trial and proposal trajectory, >= 1 (1) */
  int32_t max_search_steps;      /* step size: >= 0 (10) */
  int32_t criterion;             /* step size: BJX_GIST_SYMMETRIC (default) or BJX_GIST_ASYMMETRIC */
} bjx_gist_params;
/* Optional per-transition outputs (NULL => not written), [C] each unless marked. */
typedef struct {
  float* acceptance_rate;          /* exp(min(delta + log_ratio, 0)) */
  uint8_t* is_accepted;
  uint8_t* is_divergent;           /* -delta > divergence_threshold */
  float* energy;                   /* energy of the proposal */
  float* momentum;                 /* [C,D] momentum drawn at the start of the transition */
  int32_t* num_integration_steps;  /* steps of the proposal's own trajectory (L, or num_integration_steps) */
  int32_t* forward;                /* U (num_steps_to_uturn_forward) or j (step_index) */
  int32_t* reverse;                /* N (num_steps_to_uturn_reverse) or j_rev (reverse_step_index) */
  uint8_t* rejected;               /* is_no_return_rejected or search_exhausted */
  float* a;                        /* step size: the thresholds (a, b) and the step size used */
  float* b;
  float* step_size;
} bjx_gist_info;
/* One transition; out may alias in (in place), step_size_dev [C] overrides step_size.  Keys follow bjx_set_key_mode. */
int bjx_gist_step(bjx_handle_t h, const bjx_gist_params* params, const uint32_t* keys, const float* q_in,
                  const float* logp_in, const float* grad_in, float* q_out, float* logp_out, float* grad_out,
                  float step_size, const float* step_size_dev, const bjx_gist_info* info);
/* run_inference_algorithm (util.py:150-213) for GIST, like bjx_nuts_sample: step keys = split(rng_key, num_steps), one
 * persistent launch whose warps take whole chains through all transitions in place, bit-identical to num_steps calls of
 * bjx_gist_step; no host synchronisation.  history (optional) float32 [num_steps / thin, C, D]; acceptance_history
 * (optional) float32 [num_steps, C]; num_integration_steps_history (optional) int32 [num_steps, C]. */
int bjx_gist_sample(bjx_handle_t h, const bjx_gist_params* params, const uint32_t* rng_key, float* q, float* logp,
                    float* grad, float step_size, const float* step_size_dev, int32_t num_steps, float* history,
                    int32_t thin, float* acceptance_history, int32_t* num_integration_steps_history);

/* ---- MALA and Barker's proposal (blackjax/mcmc/mala.py, blackjax/mcmc/barker.py) ---------------------------------------
 * State (q [C,D], logp [C], grad [C,D]) as HMC's; initialise it with bjx_init_state.  One transition is one gradient
 * evaluation, a few passes over the row and one accept test: (k0, key_rmh) = split(key); accept when
 * uniform(key_rmh) < clip(exp(log_p_accept), max=1).
 *   MALA: y = x + step_size * grad + sqrt(2 step_size) * normal(k0, (D,)); log_p_accept = safe_energy_diff(E(y->x), E(x->y))
 *     with E(a->b) = -logp_b + 0.25 (1 / step_size) |a - b - step_size grad_b|^2 (NaN -> -inf).  No metric: none needs to
 *     be set, and a set one is ignored.
 *   Barker: (key_normal, key_sign) = split(k0); z = step_size * normal(key_normal), c = (M^1/2)^T grad, sign +1 with
 *     probability 1 / (1 + exp(-c z)) from uniform(split(key_sign, 1)[0], (D,)); y = x + M^1/2 (+-z); the acceptance
 *     ratio of barker.py:80-128 as written there (a NaN ratio gives acceptance_rate NaN and a rejection).  Metrics:
 *     BJX_METRIC_DIAG and BJX_METRIC_DIAG_PER_CHAIN for 1 <= dim <= 18432, BJX_METRIC_DENSE for dim <= 128 (M^1/2 =
 *     chol(M^-1)^-T); other metrics return BJX_E_UNSUPPORTED.
 * Rows: every row target and row plug-in for dim <= 1024, every big-row target and big plug-in for 1024 < dim <= 18432
 * (dim % 4 == 0).  A dense Gaussian target beyond 128 dims (the tensor-core path) returns BJX_E_UNSUPPORTED. */
typedef struct {                 /* optional per-transition outputs (NULL => not written) */
  float* acceptance_rate;        /* [C]  clip(exp(log_p_accept), max=1) */
  uint8_t* is_accepted;          /* [C] */
  float* proposal_position;      /* [C,D] the proposal, accepted or not */
  float* proposal_logdensity;    /* [C] */
  float* proposal_grad;          /* [C,D] */
} bjx_langevin_info;
/* One transition; out may alias in (in place), step_size_dev [C] overrides step_size.  Keys follow bjx_set_key_mode. */
int bjx_mala_step(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logp_in, const float* grad_in,
                  float* q_out, float* logp_out, float* grad_out, float step_size, const float* step_size_dev,
                  const bjx_langevin_info* info);
int bjx_barker_step(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logp_in, const float* grad_in,
                    float* q_out, float* logp_out, float* grad_out, float step_size, const float* step_size_dev,
                    const bjx_langevin_info* info);
/* run_inference_algorithm (util.py:150-213): step keys = split(rng_key, num_steps) on the device, then num_steps
 * transitions in place with no host synchronisation, bit-identical to num_steps step calls with those keys (shared step
 * key mode, bjx_set_key_mode's chain_offset honoured).  history (optional) float32 [num_steps / thin, C, D];
 * acceptance_history (optional) float32 [num_steps, C]. */
int bjx_mala_sample(bjx_handle_t h, const uint32_t* rng_key, float* q, float* logp, float* grad, float step_size,
                    const float* step_size_dev, int32_t num_steps, float* history, int32_t thin,
                    float* acceptance_history);
int bjx_barker_sample(bjx_handle_t h, const uint32_t* rng_key, float* q, float* logp, float* grad, float step_size,
                      const float* step_size_dev, int32_t num_steps, float* history, int32_t thin,
                      float* acceptance_history);

/* ---- Elliptical slice sampling (blackjax/mcmc/elliptical_slice.py) -------------------------------------------------------
 * State (q [C,D], logl [C]) where logl is the log-LIKELIHOOD of the handle's target; initialise it with bjx_init_state
 * (and discard the gradient row it also writes).  The Gaussian prior N(mean, cov) is set apart from the metric, and does
 * not change the route of any other call.  One transition of one chain, all in float32:
 *   (key_slice, key_momentum, key_uniform, key_theta) = split(key, 4); nu = mean + S normal(key_momentum, (D,)) with
 *   S = sqrt(cov) or chol(cov); logy = logl + log(uniform(key_uniform)); theta = 6.2831855f * uniform(key_theta), bracket
 *   [theta - 6.2831855f, theta]; p = (q - mean) cos theta + (nu - mean) sin theta + mean; subiter = 1; while
 *   logL(p) <= logy: theta = max(theta_min, f (theta_max - theta_min) + theta_min), f = uniform(fold_in(key_slice,
 *   subiter)), new p, shrink the bracket towards 0, subiter += 1.  A NaN log-likelihood ends the loop and is accepted.
 * The one deviation from the reference is the cap max_subiter (1000 in the Python API): a chain whose proposal is still
 * below the slice after max_subiter evaluations keeps (q, logl) and reports exhausted = 1, subiter = max_subiter,
 * theta = 0 and momentum = nu.  The reference would loop without end there (e.g. a start at logl = -inf); for a
 * continuous likelihood and a finite start the bracket reaches float32 resolution long before 1000 sub-iterations, so
 * the results are the reference's whenever the cap is not reached.
 * Routes (chosen from the handle):
 *   - every row target and row plug-in, 1 <= dim <= 1024, with a diagonal prior or a dense prior at dim <= 128;
 *   - a dense prior at 128 < dim <= 1024 (dim % 4 == 0): chol(cov) z is a float32-accurate tensor-core product (within
 *     about 1e-5 of the row maximum);
 *   - every big-row target and big plug-in, 1024 < dim <= 18432 (dim % 4 == 0), with a diagonal prior.
 * BJX_E_UNSUPPORTED: a dense prior beyond 1024 dims or at 128 < dim with dim % 4 != 0 (from bjx_set_elliptical_prior),
 * a dense Gaussian target beyond 128 dims (the tensor-core target path), a plug-in built without the kernels of the row
 * size, and a step or sample call before bjx_set_elliptical_prior. */
/* kind: BJX_METRIC_DIAG (cov = variances [D]) or BJX_METRIC_DENSE (cov [D, D], chol formed in float64 on the host;
 * BJX_E_INVALID when it is not positive definite).  mean [D].  Both are device arrays, copied into the handle. */
int bjx_set_elliptical_prior(bjx_handle_t h, int32_t kind, const float* mean, const float* cov);
typedef struct {            /* optional per-transition outputs (NULL => not written) */
  float* momentum;          /* [C,D] (nu - mean) cos theta - (q - mean) sin theta + mean at the accepted theta */
  float* theta;             /* [C] */
  int32_t* subiter;         /* [C] likelihood evaluations of the transition */
  uint8_t* exhausted;       /* [C] 1: max_subiter reached below the slice, state kept */
} bjx_elliptical_slice_info;
/* One transition; out may alias in (in place); max_subiter >= 1.  Keys follow bjx_set_key_mode. */
int bjx_elliptical_slice_step(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logl_in,
                              float* q_out, float* logl_out, int32_t max_subiter, const bjx_elliptical_slice_info* info);
/* run_inference_algorithm (util.py:150-213): step keys = split(rng_key, num_steps) on the device, then num_steps
 * transitions in place with no host synchronisation, bit-identical to num_steps step calls with those keys (shared step
 * key mode, bjx_set_key_mode's chain_offset honoured).  history (optional) float32 [num_steps / thin, C, D];
 * subiter_history (optional) int32 [num_steps, C]. */
int bjx_elliptical_slice_sample(bjx_handle_t h, const uint32_t* rng_key, float* q, float* logl, int32_t num_steps,
                                int32_t max_subiter, float* history, int32_t thin, int32_t* subiter_history);

/* ---- Slice sampling (blackjax/mcmc/slice.py: the multivariate slice sampler, blackjax.slice_sampling) ---------------
 * State (q [C,D], logp [C]) with logp the log-density of the handle's target; initialise it with bjx_init_state (and
 * discard the gradient row it also writes).  One transition of one chain, all in float32: (prop_key, slice_key) =
 * split(key); (level_key, interval_key, shrink_key) = split(slice_key, 3); the direction d = n / |n| with n = 0 + scale z
 * ([D] scale) or scale @ z ([D, D] scale), z = normal(prop_key, (D,)); level = logp + log(uniform(level_key)); t is in
 * the slice when logp(q + t d) >= level (q + t d unfused; a NaN log-density is never in the slice).
 *   BJX_SLICE_DOUBLING (Neal's Fig. 4 and Fig. 6): key1, key2 = split(interval_key); L0 = -width uniform(key1),
 *     R0 = L0 + width; level j widens the left end when uniform(key2, (max_expansions + 1,))[j] < 0.5, else the right
 *     one, by width 2^j; the bracket is the first level whose ends are both out of the slice, else the last, and
 *     num_expansions is its index.  A candidate must also pass the acceptance test on that bracket.
 *   BJX_SLICE_STEPPING_OUT (Fig. 3): u_key, jk_key = split(interval_key); left = -width uniform(u_key),
 *     right = left + width; j = floor(max_expansions uniform(jk_key)), k = max_expansions - 1 - j; the ends step out by
 *     width while in the slice, at most j and k times; num_expansions counts the steps.
 *   Shrinkage (Fig. 5): key = shrink_key; each try takes key, sub = split(key), t = left + uniform(sub) (right - left);
 *     found = in slice && accepted; then left = t if t < 0, right = t if t >= 0; at most max_shrinkage tries.  A chain
 *     that finds no point keeps (q, logp) bit for bit and reports is_accepted = 0.
 * The device evaluates the target fewer times than the reference (the doubling levels one at a time up to the first
 * whose ends are both out, one point per bisection of the acceptance test, the test only for candidates in the slice)
 * and decides the same.  The one deviation: the acceptance test stops after max_expansions + 1 bisections and returns
 * its verdict as it stands; that binds only when width 2^j overflowed to inf, where the reference never stops.
 * width: a scalar (> 0 and finite) or width_dev [C] per chain (then width is ignored).
 * Routes (chosen from the handle):
 *   - every row target and row plug-in, 1 <= dim <= 1024, with a [D] scale, or a [D, D] scale at dim <= 128;
 *   - every big-row target and big plug-in, 1024 < dim <= 18432 (dim % 4 == 0), with a [D] scale.
 * BJX_E_UNSUPPORTED: a dense scale beyond 128 dims (from bjx_set_slice_direction_scale), a dense Gaussian target beyond
 * 128 dims (the tensor-core target path), a plug-in built without the kernels of the row size, and a step or sample
 * call before bjx_set_slice_direction_scale.  BJX_E_INVALID: a bad width, a negative cap or an unknown interval. */
#define BJX_SLICE_DOUBLING 0
#define BJX_SLICE_STEPPING_OUT 1
/* kind: BJX_METRIC_DIAG (scale [D]) or BJX_METRIC_DENSE (scale [D, D], row-major).  A device array, copied into the
 * handle. */
int bjx_set_slice_direction_scale(bjx_handle_t h, int32_t kind, const float* scale);
typedef struct {            /* optional per-transition outputs (NULL => not written) */
  uint8_t* is_accepted;     /* [C] 1: shrinkage found a point within max_shrinkage tries */
  int32_t* num_expansions;  /* [C] */
  int32_t* num_shrink;      /* [C] shrinkage tries */
  float* bracket_left;      /* [C] the bracket in t (the current point at t = 0) */
  float* bracket_right;     /* [C] */
} bjx_slice_info;
/* One transition; out may alias in (in place).  Keys follow bjx_set_key_mode. */
int bjx_slice_step(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logp_in, float* q_out,
                   float* logp_out, float width, const float* width_dev, int32_t interval, int32_t max_expansions,
                   int32_t max_shrinkage, const bjx_slice_info* info);
/* run_inference_algorithm (util.py:150-213): step keys = split(rng_key, num_steps) on the device, then num_steps
 * transitions in place with no host synchronisation, bit-identical to num_steps step calls with those keys (shared step
 * key mode, bjx_set_key_mode's chain_offset honoured).  history (optional) float32 [num_steps / thin, C, D];
 * num_expansions_history and num_shrink_history (optional) int32 [num_steps, C]; evaluations (optional) one device
 * uint64 to which the target evaluations of the call are added. */
int bjx_slice_sample(bjx_handle_t h, const uint32_t* rng_key, float* q, float* logp, int32_t num_steps, float width,
                     const float* width_dev, int32_t interval, int32_t max_expansions, int32_t max_shrinkage,
                     float* history, int32_t thin, int32_t* num_expansions_history, int32_t* num_shrink_history,
                     uint64_t* evaluations);

/* ---- Random-walk Metropolis (blackjax/mcmc/random_walk.py: blackjax.additive_step_random_walk, rmh, irmh) -----------
 * State (q [C,D], logp [C]) with logp the log-density of the handle's target; initialise it with bjx_init_state (and
 * discard the gradient row it also writes).  The stored logp is used as given, never re-evaluated.  One transition of one
 * chain, all in float32: (key_proposal, key_accept) = split(key); z = normal(key_proposal, (D,)); lin = sigma z ([D]
 * sigma) or sigma @ z ([D, D] sigma); the proposal is y = q + lin (BJX_RW_ADDITIVE) or y = mean + lin
 * (BJX_RW_INDEPENDENT); with E(a, b) = -logp(b) - f(b, a), log_p_accept = E(y, x) - E(x, y) (NaN -> -inf),
 * acceptance_rate = min(1, exp(log_p_accept)) and the proposal is accepted when uniform(key_accept) < acceptance_rate.
 * f = 0 unless correct != 0; then f(b, a) = -0.5 sum ((a - mean) / sigma)^2, the log-density of the independent proposal
 * N(mean, diag(sigma)^2) at a without its constant terms (they cancel).  A rejected chain keeps (q, logp) bit for bit.
 * Routes (chosen from the handle):
 *   - every row target and row plug-in, 1 <= dim <= 1024, with a [D] sigma, or a [D, D] sigma at dim <= 128;
 *   - every big-row target and big plug-in, 1024 < dim <= 18432 (dim % 4 == 0), with a [D] sigma.
 * BJX_E_UNSUPPORTED: a dense sigma beyond 128 dims (from bjx_set_rw_proposal), a dense Gaussian target beyond 128 dims
 * (the tensor-core target path), a plug-in built without the kernels of the row size, a step or sample call before
 * bjx_set_rw_proposal, and correct != 0 with a dense sigma or an additive proposal. */
#define BJX_RW_ADDITIVE 0
#define BJX_RW_INDEPENDENT 1
/* kind: BJX_RW_ADDITIVE (mean NULL) or BJX_RW_INDEPENDENT (mean [D]); sigma_kind: BJX_METRIC_DIAG (sigma [D]) or
 * BJX_METRIC_DENSE (sigma [D, D], row-major, dim <= 128).  Device arrays, copied into the handle. */
int bjx_set_rw_proposal(bjx_handle_t h, int32_t kind, const float* mean, int32_t sigma_kind, const float* sigma);
typedef struct {            /* optional per-transition outputs (NULL => not written) */
  float* acceptance_rate;   /* [C] */
  uint8_t* is_accepted;     /* [C] */
} bjx_rw_info;
/* One transition; out may alias in (in place, both of (q, logp)).  Keys follow bjx_set_key_mode. */
int bjx_rw_step(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logp_in, float* q_out,
                float* logp_out, int32_t correct, const bjx_rw_info* info);
/* run_inference_algorithm (util.py:150-213): step keys = split(rng_key, num_steps) on the device, then num_steps
 * transitions in place with no host synchronisation, bit-identical to num_steps step calls with those keys (shared step
 * key mode, bjx_set_key_mode's chain_offset honoured).  history (optional) float32 [num_steps / thin, C, D];
 * acceptance_history (optional) float32 [num_steps, C]. */
int bjx_rw_sample(bjx_handle_t h, const uint32_t* rng_key, float* q, float* logp, int32_t num_steps, int32_t correct,
                  float* history, int32_t thin, float* acceptance_history);

/* ---- Adjusted MCLMC tuning: adjusted_mclmc_find_L_and_step_size (blackjax/adaptation/adjusted_mclmc_adaptation.py:26-507)
 * Every chain runs the reference's single-chain tuner with its own key, as jax.vmap over chains would, and ends with its own
 * (L, step_size, inverse_mass_matrix).  Supported configurations are those of bjx_adjusted_mclmc_step (BJX_E_UNSUPPORTED
 * otherwise).  The kernel being tuned is adjusted_mclmc (random_generator_arg NULL: ceil(L / step_size) steps, reported as
 * the float L / step_size) or adjusted_mclmc_dynamic (random_generator_arg [C, 2], advanced in place, with steps_rule and
 * min_steps as in bjx_adjusted_mclmc_sample and avg = L / step_size per chain); L_proposal_factor is inf. */
/* One tuning step (dual_avg_step, adjusted_mclmc_adaptation.py:236-311) in place, for every chain.  keys (per
 * bjx_set_key_mode) drive one transition with the handle's metric at avg = L / step_size.  A chain whose output position is
 * not finite keeps its whole previous state, random_generator_arg included; otherwise its state is nan_to_num of the new
 * one (a rejected transition leaves the stored rows as they are).  da_state [C, 5] (log_step, log_step_avg, step,
 * avg_error, mu) takes one dual-averaging update on the acceptance rate toward target, kept only where mask = 1; then
 * step = clamp(1e-5, exp(log_step), L / 1.1) and log_step = log(step).  With mask = 0, total [C] and moments [C, 2, D]
 * (16-byte aligned) take the streaming average of (x, x^2) with weight success * step (incremental_value_update,
 * util.py:291-319); with mask = 1 they are not touched (the reference's update is the identity there for total = 0).  With
 * mask = 1 step_size becomes step and, unless fix_L, L becomes L * (step / old step size).  count [C] (optional) adds the
 * transition's num_integration_steps.  success (optional) [C] uint8: the output position was finite; steps (optional) [C]
 * int32: the integration steps run. */
int bjx_adjusted_mclmc_tune_step(bjx_handle_t h, const uint32_t* keys, float* q, float* logp, float* grad,
                                 uint32_t* random_generator_arg, int32_t steps_rule, int32_t min_steps, float* step_size,
                                 float* L, float* da_state, float* total, float* moments, float* count, int32_t mask,
                                 int32_t fix_L, float target, uint8_t* success, int32_t* steps);
/* adjusted_mclmc_find_L_and_step_size, all windows and stages on the handle's stream with no host synchronisation.  rng_key
 * per bjx_set_key_mode: one key [2] (chain c: split(rng_key, n_global)[chain_offset + c]) or per-chain keys [C, 2].  The
 * host computes the stage lengths after frac /= num_windows: num_steps1 = int(N frac_tune1), num_steps2 = int(N frac_tune2),
 * num_steps3 = int(N frac_tune3) or 0 when frac_tune3 = 0.  step_size [C], L [C] and inverse_mass_matrix [C, D] (a per-chain
 * diagonal metric, used in place of the handle's, which must still be a diagonal kind) are the initial parameters in and
 * the tuned ones out; L enters and leaves pinned to target_num_integration_steps * step_size.  Each window runs pass 1
 * (num_steps1 + num_steps2 tuning steps, L fixed, the moments over the last num_steps2), and if num_steps2 != 0 the
 * variance step (L and step_size scaled by clamp(0, contract(var) / L, 2), contract = sqrt(sum var) * tuning_factor, or
 * sqrt(max var * D) * tuning_factor with use_max; inverse_mass_matrix = var with diagonal_preconditioning) and pass 2
 * (num_steps1 steps, L tracking the step size).  If num_steps3 >= 2, each window then runs num_steps3 transitions and sets
 * L = min(l_factor * L / r, 2 L) with r the per-chain ESS (mean over dimensions, or min with use_max) per transition, on
 * slices of chains whose history [num_steps3, slice, D] fits max_history_bytes (at least one chain; the result does not
 * depend on the slice size), followed by a pass 1 with num_steps2 = 0.  num_integration_steps [C] receives the summed
 * num_integration_steps of every tuning transition. */
int bjx_adjusted_mclmc_find_l_and_step_size(bjx_handle_t h, const uint32_t* rng_key, float* q, float* logp, float* grad,
                                            uint32_t* random_generator_arg, int32_t steps_rule, int32_t min_steps,
                                            float* step_size, float* L, float* inverse_mass_matrix, int32_t num_windows,
                                            int32_t num_steps1, int32_t num_steps2, int32_t num_steps3, float target,
                                            int32_t diagonal_preconditioning, int32_t use_max, float tuning_factor,
                                            float target_num_integration_steps, double l_factor, int64_t max_history_bytes,
                                            float* num_integration_steps);

/* ---- LAPS: the ensemble MCLMC warm-up (blackjax/adaptation/laps.py, laps_burn_in.py, eca.py) -------------------------
 * One shared (step size, L, diagonal metric) for all chains of the handle, updated after every step from ensemble averages.
 * state is a caller-owned float32 buffer of bjx_laps_state_floats(n_chains, dim, save_num, equi_full) floats (16-byte
 * aligned) that carries the adaptation state and the scratch of both phases; save_num = rint(save_frac * num_steps1) >= 1.
 * Every call on one state must pass the save_num it was sized with, and its burn-in steps the sizing's equi_full.
 * phase_key is a HOST pointer to one raw key [2] (the phase's key1 / key2): chain c at step t uses
 * fold_in(fold_in(key, 0), (chain_offset + c) T + t), equipartition_fullrank's probes fold_in(fold_in(key, 1), t).  The
 * handle's metric must be the identity during the burn-in and the metric of the adjusted phase afterwards (the state's
 * M^-1 = floats [16, 16 + dim), or ones), a shared diagonal metric [dim].  Supported configurations are those of
 * bjx_mclmc_step with that metric kind (BJX_E_UNSUPPORTED otherwise). */
typedef struct {
  int32_t save_num;    /* rows of the history ring */
  float alpha, C, r_end;
  int32_t bias_type;   /* 0 r_max, 1 r_avg, 2 equi_full, 3 equi_diag */
  int32_t early_stop;
  int32_t equi_full;   /* compute equipartition_fullrank (required by bias_type 2) */
} bjx_laps_burn_in_config;
int64_t bjx_laps_state_floats(int32_t n_chains, int32_t dim, int32_t save_num, int32_t equi_full);
/* laps_burn_in.initialize after sample_init: logp, grad = value_and_grad(q); u = grad / |grad| with dimension i's sign
 * flipped when mean_c(-x_i g_i) < 1; the burn-in's initial adaptation state (L = inf, step size 0.01 sqrt(dim)). */
int bjx_laps_init(bjx_handle_t h, const float* q, float* logp, float* grad, float* u, float* state, int32_t save_num);
/* Burn-in step t of num_steps in place on (q, u, logp, grad, state): one fused MCLMC transition with nan_reject and the
 * per-CTA sums, their merge, equipartition_fullrank if asked, and Adaptation.update with the stop rule.  info (optional,
 * device, [num_steps, 9]) row t receives (L, step_size, EEVPD_wanted, EEVPD, equi_diag, equi_full, r_max, r_avg, entropy).
 * After the stop every launch returns at once. */
int bjx_laps_burn_in_step(bjx_handle_t h, const uint32_t* phase_key, int32_t t, int32_t num_steps, float* q, float* u,
                          float* logp, float* grad, float* state, const bjx_laps_burn_in_config* cfg, float* info);
/* All num_steps burn-in steps, reading the device's stop flag once per `chunk` steps (the result does not depend on chunk);
 * *steps_run (host) receives the number of steps taken. */
int bjx_laps_burn_in_run(bjx_handle_t h, const uint32_t* phase_key, int32_t num_steps, float* q, float* u, float* logp,
                         float* grad, float* state, const bjx_laps_burn_in_config* cfg, float* info, int32_t chunk,
                         int32_t* steps_run);
/* laps.py:250-257: with diagonal_preconditioning, step size /= sqrt(mean(M^-1)); the bisection starts at [-inf, inf]. */
int bjx_laps_switch(bjx_handle_t h, float* state, int32_t diagonal_preconditioning);
/* Adjusted step t of num_samples in place on (q, logp, grad, state): one static adjusted MCLMC transition
 * (steps_per_sample steps, L_proposal_factor 1.25, the state's step size, the handle's metric and integrator), the ensemble
 * mean acceptance and bisection_monotonic_fn(target_acceptance).  info (optional, device, [num_samples, 4]) row t receives
 * (L = step_size steps_per_sample, step_size, acc_prob, equi_diag); equi_diag is NaN and skipped without diagnostics. */
int bjx_laps_adjusted_step(bjx_handle_t h, const uint32_t* phase_key, int32_t t, int32_t num_samples, float* q, float* logp,
                           float* grad, float* state, int32_t save_num, int32_t steps_per_sample, float target_acceptance,
                           int32_t diagnostics, float* info);
int bjx_laps_adjusted_run(bjx_handle_t h, const uint32_t* phase_key, int32_t num_samples, float* q, float* logp,
                          float* grad, float* state, int32_t save_num, int32_t steps_per_sample, float target_acceptance,
                          int32_t diagnostics, float* info);

/* ---- PRNG (jax.random restated; keys raw uint32 pairs) ----------------------------------------- */
/* h may be NULL for the PRNG entry points: current device, and the stream this thread registered with
 * bjx_set_default_stream (a cudaStream_t; the legacy default stream until one is registered) */
int bjx_set_default_stream(void* cuda_stream);
int bjx_prng_split(bjx_handle_t h, const uint32_t* keys, int64_t n_keys, int32_t num, uint32_t* out);
int bjx_prng_fold_in(bjx_handle_t h, const uint32_t* keys, int64_t n_keys, uint32_t data, uint32_t* out);
int bjx_prng_random_bits(bjx_handle_t h, const uint32_t* keys, int64_t n_keys, int64_t per_key, uint32_t* out);
int bjx_prng_uniform(bjx_handle_t h, const uint32_t* keys, int64_t n_keys, int64_t per_key, float* out);
int bjx_prng_normal(bjx_handle_t h, const uint32_t* keys, int64_t n_keys, int64_t per_key, float* out);
/* jax.random.randint(key, shape, minval, maxval) int32 -- dynamic_hmc's default integration_steps_fn
 * (dynamic_hmc.py:66: randint(key, (), 1, 10)) */
int bjx_prng_randint(bjx_handle_t h, const uint32_t* keys, int64_t n_keys, int64_t per_key, int32_t minval, int32_t maxval,
                     int32_t* out);

/* ---- window adaptation (staged_adaptation.py:111-307) -------------------------------------------- */
/* Per-chain dual averaging (optimizers/dual_averaging.py:87-129).  da_state float32 [C,5] =
 * (log_step, log_step_avg, step, avg_error, mu).  step_size_out [C] = exp(log_step). */
int bjx_da_init(bjx_handle_t h, float* da_state, const float* initial_step_size /*[C]*/, float* step_size_out);
int bjx_da_update(bjx_handle_t h, float* da_state, const float* acceptance_rate, float target, float* step_size_out);
/* slow-window end: re-initialise DA at exp(log_step_avg) (staged_adaptation.py:233-249) */
int bjx_da_reset(bjx_handle_t h, float* da_state, float* step_size_out);
int bjx_da_final(bjx_handle_t h, const float* da_state, float* step_size_out);
/* Per-chain diagonal Welford (adaptation/mass_matrix.py:411-442): mean,m2 [C,D]; count is a host int */
int bjx_welford_update(bjx_handle_t h, const float* q, float* mean, float* m2, int32_t new_count);
/* regularised IMM (mass_matrix.py:335-357): imm = n/(n+5) m2/(n-1) + 1e-3*5/(n+5); resets mean,m2 */
int bjx_welford_final(bjx_handle_t h, float* mean, float* m2, int32_t count, float* imm_out);
/* Per-chain dense Welford (mass_matrix.py:411-442 with is_diagonal_matrix=False): mean [C,D], m2 [C,D,D];
 * m2 += outer(x - mean_new, x - mean_old) */
int bjx_welford_dense_update(bjx_handle_t h, const float* q, float* mean, float* m2, int32_t new_count);
/* regularised dense IMM per chain (mass_matrix.py:335-357): imm = n/(n+5) m2/(n-1) + 1e-3*5/(n+5) I; resets mean,m2 */
int bjx_welford_dense_final(bjx_handle_t h, float* mean, float* m2, int32_t count, float* imm_out);
/* Chain-pooled summary block of THIS GPU's chains for the shared-epsilon warm-up
 * (staged_adaptation.py:153-171,906-966; metric_buffers.py:396-420):
 * stats_out float32 [2 + 2*D] = (sum acceptance_rate, n_chains, mean[D], M2[D]).
 * The blocks of all GPUs are exchanged with ONE all-gather and CGL-merged on every rank. */
int bjx_pooled_stats(bjx_handle_t h, const float* q, const float* acceptance_rate, float* stats_out);
/* Dense variant (welford_dense recipe; metric_buffers.py:396-420 `centered.T @ centered`), any dim (float32 SIMT tiles in
 * a fixed order; dim = 512 x 32768 chains: a few ms):
 * stats_out float32 [2 + D + D*D] = (sum acceptance_rate, n_chains, mean[D], M2[D,D]). */
int bjx_pooled_stats_dense(bjx_handle_t h, const float* q, const float* acceptance_rate, float* stats_out);

/* ---- shared (cross-chain, cross-GPU) window adaptation, device resident ------------------------------------------
 * The reference's multi-chain path (staged_adaptation.py:153-171,906-966): ONE dual-averaging update per warm-up step
 * on the mean acceptance rate of ALL chains and, in slow windows, the chain-pooled moment block merged into the window
 * accumulator (metric_buffers.py:334-420); its cross-device collective is lax.psum over "chains" (eca.py:56-62).
 * Here: each GPU reduces its chains in fixed blocks of BJX_STAT_BLOCK_CHAINS chains to (sum accept, n, mean[D], M2[D]),
 * ONE NCCL all-gather exchanges the blocks, and every rank merges them in global chain order and applies the same
 * update on the device -- results do not depend on the GPU count when chains_per_gpu % BJX_STAT_BLOCK_CHAINS == 0. */
#define BJX_STAT_BLOCK_CHAINS 4096
/* NCCL communicator helpers (libnccl.so.2 is bound at run time; single-GPU callers never need it).  A caller that
 * already owns an ncclComm_t (e.g. an XLA / framework communicator) passes it to the calls below as is. */
int bjx_nccl_unique_id(void* id128_out);                      /* ncclGetUniqueId: 128 bytes, on rank 0 */
int bjx_nccl_comm_init_rank(const void* id128, int32_t n_ranks, int32_t rank, int32_t device, void** nccl_comm_out);
int bjx_nccl_comm_destroy(void* nccl_comm);
/* The collective of the path: all-gather `count` floats per rank into gathered[n_ranks * count] on the handle's stream.
 * nccl_comm is an ncclComm_t (NULL: one rank, gathered = block). */
int bjx_allgather_stats(bjx_handle_t h, void* nccl_comm, const float* block, int64_t count, float* gathered);
/* Device state of the shared adaptation: bjx_adapt_shared_state_floats(...) floats (dual averaging, window accumulator,
 * this rank's blocks and the gathered blocks). */
int64_t bjx_adapt_shared_state_floats(int32_t n_chains_local, int32_t dim, int32_t n_ranks);
/* step_size_chain_out [C] (every entry = initial_step_size: the array the transition kernels read as per-chain step
 * sizes), imm_out [D] = ones (also installed as the handle's diagonal metric). */
int bjx_adapt_shared_init(bjx_handle_t h, float* state, float initial_step_size, float* step_size_chain_out, float* imm_out);
/* One warm-up step after the transition: block statistics of (q, acceptance_rate) -> all-gather -> merge, dual
 * averaging, window bookkeeping (stage: 0 fast / 1 slow; window_end: last step of a slow window: imm rewritten,
 * accumulator reset, dual averaging re-initialised, the handle's metric re-installed).  step_size_chain [C] is
 * refilled with the new step size.  eps_history (nullable, device): the step size of warm-up step t lands in [t].
 * Fully asynchronous on the handle's stream. */
int bjx_adapt_shared_update(bjx_handle_t h, void* nccl_comm, int32_t n_ranks, float* state, const float* q,
                            const float* acceptance_rate, int32_t stage, int32_t window_end, float target_acceptance,
                            float* step_size_chain, float* imm, float* eps_history);
/* The whole shared warm-up as one call (staged_adaptation.py:906-966): for t < num_steps one in-place transition with step
 * key split(rng_key, num_steps)[t] (NUTS when max_num_doublings > 0, else HMC with num_integration_steps) followed by
 * bjx_adapt_shared_update with schedule[t] = stage | window_end << 1 (HOST array, staged_adaptation.py:315-405).
 * state / step_size_chain / imm as initialised by bjx_adapt_shared_init; acceptance_scratch: device float32 [C];
 * steps_scratch (device int32 [C]) + leapfrog_counter (device uint64, caller-zeroed): optional, the executed leapfrogs
 * summed over chains and steps.  Asynchronous: the loop only enqueues. */
int bjx_adapt_shared_run(bjx_handle_t h, void* nccl_comm, int32_t n_ranks, const uint32_t* rng_key, const uint8_t* schedule,
                         int32_t num_steps, float* q, float* logp, float* grad, float* state, float* step_size_chain,
                         float* imm, float target_acceptance, int32_t max_num_doublings, int32_t num_integration_steps,
                         float* eps_history, float* acceptance_scratch, int32_t* steps_scratch,
                         unsigned long long* leapfrog_counter);
/* final step size exp(log_step_avg) (staged_adaptation.py:303) into step_size_out [1] (device) */
int bjx_adapt_shared_final(bjx_handle_t h, const float* state, float* step_size_out);

/* ---- Low-rank window adaptation (low_rank_adaptation.py:458-652, buffer_policy="reset"), pooled over chains ----------
 * ONE step size and ONE low-rank metric M^-1 = diag(sigma) (I + U (diag(lam) - I) U^T) diag(sigma) for all C chains of one
 * GPU, adapted by Stan's window schedule with the Fisher-divergence estimator (_compute_low_rank_metric,
 * metric_estimators.py:618-808) at every window end.  The handle must hold a rank-k low-rank metric (k = max_rank,
 * bjx_set_metric_low_rank); the warm-up rewrites its block in place on the stream.  Built for dim <= 512 and 1 <= k <= 16
 * on the warp kernels; otherwise BJX_E_UNSUPPORTED.
 * state float32 [bjx_lowrank_window_state_floats(C, D, k)]; its first 64 floats are
 *   [0..7] the dual-averaging slots of bjx_adapt_shared_* ([5] the current step size, [7] steps taken)
 *   [8] slow steps of the current window   [9] windows ended
 *   [32..48) and [48..64) the eigensolver headers of the draws' and the gradients' top-k solves, slots as in
 *   bjx_meads_lrd_state_floats ([1] iterations of the last solve, [2] its largest relative residual, [3] sticky
 *   non-converged flag, [4] sum and [5] maximum of the iterations, [6] solves)
 * followed by sigma[D] | U[D,k] | lam[k] | mu*[D], the metric of the last window end (initially ones, zeros, ones, zeros).
 * bjx_lowrank_window_init: zero-fills the state, initialises dual averaging at initial_step_size (step_size_chain_out [C]
 * filled with it) and installs the initial metric.
 * bjx_lowrank_window_update: one warm-up step after the transition.  schedule = stage | window_end << 1 | retained << 2:
 * dual averaging on the mean of acceptance_rate [C] every step; on a retained slow step q and grad [C, D] are folded into
 * the windowed accumulators of the draws and the gradients; every slow step counts towards the window's n = C x steps;
 * at a window end (a retained slow step) the estimator runs with gamma and cutoff, the metric is re-installed, the
 * accumulators are reset and dual averaging restarts at exp(log_step_avg).  Retain the last min(steps, B) steps of every
 * window to reproduce the reference's circular buffer of B steps.  eps_history (nullable, device): step size of step t.
 * bjx_lowrank_window_run: the whole warm-up as one call, the loop of bjx_adapt_shared_run with this update.
 * bjx_lowrank_window_final: step_size_out [1] = exp(log_step_avg), mu_star_out [D], sigma_out [D], U_out [D,k],
 * lam_out [k] (device).  Every reduction has a fixed order: two runs are bit-identical. */
size_t bjx_lowrank_window_state_floats(int32_t n_chains, int32_t dim, int32_t rank);
int bjx_lowrank_window_init(bjx_handle_t h, float* state, float initial_step_size, float* step_size_chain_out);
int bjx_lowrank_window_update(bjx_handle_t h, float* state, const float* q, const float* grad, const float* acceptance_rate,
                              int32_t schedule, float target_acceptance, float gamma, float cutoff, float* step_size_chain,
                              float* eps_history);
int bjx_lowrank_window_run(bjx_handle_t h, const uint32_t* rng_key, const uint8_t* schedule, int32_t num_steps, float* q,
                           float* logp, float* grad, float* state, float* step_size_chain, float target_acceptance,
                           float gamma, float cutoff, int32_t max_num_doublings, int32_t num_integration_steps,
                           float* eps_history, float* acceptance_scratch, int32_t* steps_scratch,
                           unsigned long long* leapfrog_counter);
int bjx_lowrank_window_final(bjx_handle_t h, const float* state, float* step_size_out, float* mu_star_out, float* sigma_out,
                             float* U_out, float* lam_out);

/* ---- ChEES-HMC warm-up (blackjax/adaptation/chees_adaptation.py, mass_matrix_estimation=None; SURVEY 8f item 4) --------------
 * Cross-chain adaptation of the step size (dual averaging on the harmonic mean of the acceptance probabilities) and of the
 * trajectory length (Adam on log T along the ChEES gradient), device resident, two all-gathers of block statistics per
 * step.  The transition is an HMC step with per-chain arrays the update rewrites: step_size_chain [C] (one value) and
 * steps_chain int32 [C] = ceil(jitter(i) * T / eps) with the base-2 Halton jitter (dynamic_hmc.py:205-215); pass the
 * latter to bjx_set_integration_steps and request proposal_position / proposal_momentum in bjx_info. */
int64_t bjx_chees_state_floats(int32_t n_chains_local, int32_t dim, int32_t n_ranks);
int bjx_chees_init(bjx_handle_t h, float* state, float step_size, int32_t max_bits, float jitter_amount,
                   float* step_size_chain_out, int32_t* steps_chain_out);
/* one warm-up step after the transition; optimiser = Adam(learning_rate, b1, b2, eps 1e-8); history (nullable, device
 * [num_steps, 4]) receives (step_size, trajectory_length, next step count, ChEES gradient) */
int bjx_chees_update(bjx_handle_t h, void* nccl_comm, int32_t n_ranks, float* state, const float* initial_position,
                     const float* proposal_position, const float* proposal_momentum, const float* acceptance_rate,
                     const uint8_t* is_divergent, float learning_rate, float b1, float b2, float target_acceptance,
                     float decay_rate, int32_t max_leapfrog_steps, float* step_size_chain, int32_t* steps_chain, float* history);
/* out2 (HOST, 2 floats): step_size = exp(log_step_size_moving_average), num_leapfrog_steps = exp(log T_ma - log eps_ma);
 * synchronises the stream */
int bjx_chees_final(bjx_handle_t h, const float* state, float* out2_host);

/* ---- ChEES with an ensemble-estimated diagonal metric (chees_adaptation.py:61-237,797-1001, mass_matrix_estimation=
 * "diagonal") ----------------------------------------------------------------------------------------------------------------
 * Same step as bjx_chees_update plus: in-window steps fold the new positions (after the transition) of all chains of all
 * ranks into a diagonal accumulator (pooled in BJX_STAT_BLOCK_CHAINS blocks, carried by the step's first all-gather) and
 * rewrite imm [D] = max(m2 / (n - 1), 1e-20) once n >= max(64, int(2 sqrt(D))), ones before that; the handle's metric is
 * re-installed on the stream.  options: BJX_CHEES_WHITEN whitens the criterion by imm; BJX_CHEES_LENGTH_FLOOR also keeps a
 * windowed D x D covariance accumulator per block, refreshes lambda_max (top eigenvalue of the imm-whitened covariance, 5
 * power iterations) on steps with `recompute`, and the next transition consumes min(max(T, (pi/2) sqrt(lambda_max)),
 * max_leapfrog_steps * eps) once imm is engaged.  dim <= 1024.  `state` is a bjx_chees_state_floats buffer initialised
 * by bjx_chees_init, metric_state a bjx_chees_metric_state_floats buffer initialised by bjx_chees_metric_init (which
 * sets imm_out to ones and installs it).  lambda_history / engaged_history (nullable, device [num_steps]): lambda_max and
 * the engagement flag after step t, i.e. those the transition of step t + 1 uses. */
#define BJX_CHEES_WHITEN 1
#define BJX_CHEES_LENGTH_FLOOR 2
int64_t bjx_chees_metric_state_floats(int32_t n_chains_local, int32_t dim, int32_t n_ranks, int32_t options);
int bjx_chees_metric_init(bjx_handle_t h, float* metric_state, int32_t n_ranks, int32_t options, float* imm_out);
int bjx_chees_update_metric(bjx_handle_t h, void* nccl_comm, int32_t n_ranks, int32_t options, float* state,
                            float* metric_state, const float* initial_position, const float* proposal_position,
                            const float* proposal_momentum, const float* new_position, const float* acceptance_rate,
                            const uint8_t* is_divergent, float learning_rate, float b1, float b2, float target_acceptance,
                            float decay_rate, int32_t max_leapfrog_steps, int32_t in_window, int32_t recompute,
                            float* step_size_chain, int32_t* steps_chain, float* history, float* imm, float* lambda_history,
                            float* engaged_history);
/* out4 (HOST): step_size, num_leapfrog_steps (with the floor re-applied after 20 power iterations against imm),
 * floor_clipped_by_cap (0 / 1), lambda_max; synchronises the stream */
int bjx_chees_final_metric(bjx_handle_t h, void* nccl_comm, int32_t n_ranks, int32_t options, const float* state,
                           float* metric_state, int32_t max_leapfrog_steps, const float* imm, float* out4_host);
/* Fold positions q [C, D] (device) into this rank's windowed covariance accumulators, as an in-window step does
 * (needs BJX_CHEES_LENGTH_FLOOR). */
int bjx_chees_metric_fold_covariance(bjx_handle_t h, int32_t options, float* metric_state, const float* q);
/* The accumulators merged over all ranks: out (device) = (count, mean[D], covariance m2 / max(count - 1, 1) [D, D]). */
int bjx_chees_metric_covariance(bjx_handle_t h, void* nccl_comm, int32_t n_ranks, int32_t options, float* metric_state,
                                float* out);

/* ---- diagnostics on a device-resident history (SURVEY 8f item 3) ---------------------------------------------- */
/* blackjax.diagnostics.potential_scale_reduction (diagnostics.py:39-89): history float32 [num_samples, C, D] as written
 * by bjx_hmc_sample; rhat_out float32 [D]; scratch: at least 2*C*D + 4 + 4*D floats (device). */
int bjx_potential_scale_reduction(bjx_handle_t h, const float* history, int32_t num_samples, float* rhat_out,
                                  float* scratch);

/* blackjax.diagnostics.effective_sample_size (diagnostics.py:159-305; Geyer initial positive + monotone sequences on
 * the chain-averaged autocovariance), same history layout; ess_out float32 [D]; scratch: 8-byte aligned device buffer of
 * at least bjx_ess_scratch_floats(num_samples, C, D) floats.  One chain is allowed (no between-chain term). */
int64_t bjx_ess_scratch_floats(int32_t num_samples, int32_t n_chains, int32_t dim);
int bjx_effective_sample_size(bjx_handle_t h, const float* history, int32_t num_samples, float* ess_out, float* scratch);

/* Rank-normalised split diagnostics (blackjax/diagnostics.py:92-155, 341-522; Vehtari et al. 2021) over the same history
 * layout.  Each chain is split into halves of h = num_samples / 2 draws (an odd last draw is dropped), giving 2C chains;
 * every dimension's n = 2C * h pooled draws are ranked with ties broken by pooled index (-0 == +0, NaN after +inf) and
 * scored z = Phi^-1((r - 3/8) / (n + 1/4)) in float64.  Dimensions are processed dims_per_pass at a time: the calls take
 * the largest pass width whose scratch fits scratch_bytes (a multiple of 32 when that leaves at least 32).
 * Rejected with BJX_E_INVALID: num_samples < 4, n >= 2^31, a scratch buffer too small for one dimension per pass, a
 * scratch pointer not 256-byte aligned.  No host synchronisation. */
int64_t bjx_rank_diagnostics_scratch_bytes(int32_t num_samples, int32_t n_chains, int32_t dim, int32_t dims_per_pass);
/* out float32 [h, 2C, D]: the rank-normalised split draws, or with folded != 0 those of |x - median| */
int bjx_rank_normalize(bjx_handle_t h, const float* history, int32_t num_samples, int32_t folded, float* out,
                       void* scratch, size_t scratch_bytes);
/* rhat_out = max(R-hat of the scores, R-hat of the folded scores), ess_bulk_out = ESS of the scores, ess_tail_out =
 * min(ESS of 1[x <= q_lo], ESS of 1[x >= q_hi]) with q_lo, q_hi the pooled linear quantiles at (1 -+ prob) / 2; each
 * float32 [D], NULL skips its work.  A column with a NaN draw reports NaN in all three.  prob in (0, 1). */
int bjx_rank_diagnostics(bjx_handle_t h, const float* history, int32_t num_samples, double prob, float* rhat_out,
                         float* ess_bulk_out, float* ess_tail_out, void* scratch, size_t scratch_bytes);

#ifdef __cplusplus
}
#endif
#endif /* BJX_H_ */
