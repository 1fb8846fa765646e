"""Restatement of BlackJAX's ChEES-HMC warm-up (Halton jitter; identity metric, or mass_matrix_estimation="diagonal":
the ensemble-estimated diagonal inverse mass matrix, the whitened ChEES criterion and the slow-direction trajectory-length
floor).

TEST INFRASTRUCTURE (see oracle/__init__.py).  float32.

Follows blackjax/adaptation/chees_adaptation.py:
* state / init             :28-58, :513-523
* compute_parameters       :307-511 (harmonic-mean dual averaging, weighted proposal mean, the ChEES gradient
                           jitter * T * (|dx'|^2 - |dx|^2) <dx', p'>, Adam on log T with the +-0.35 clip, moving averages)
* whitened criterion       :449-466
* engagement threshold     :61-72 max(64, int(2 sqrt(D)))
* engaged-or-ones metric   :75-90 max(m2 / (n - 1), 1e-20) once n >= threshold
* power iteration          :147-166 warm-started, norm guarded to 1 when 0, Rayleigh quotient
* recompute                :169-189 covariance m2 / max(count - 1, 1), whitened by 1/sqrt(imm) on both sides
* length floor             :192-236 min(max(T, (pi/2) sqrt(lambda_max)), max_leapfrog_steps * eps) when engaged
* run loop                 :737-1025 (jitter_gn, integration_steps_fn, one_step, final parameters; with the diagonal
                           metric the window starts at int(fraction * num_steps) and the eigenvalue is recomputed when
                           t % 32 == 0 in the window)
* Halton sequence          blackjax/mcmc/dynamic_hmc.py:205-215 (adjusted_mclmc.halton_sequence)
* dual averaging           blackjax/optimizers/dual_averaging.py:87-129 (gradient passed directly)
* Adam                     optax.adam(learning_rate, b1, b2, eps=1e-8): scale_by_adam with bias correction, then -lr
                           (optax is a third-party dependency of the reference, absent from /root/reference; algorithm
                           as published: Kingma & Ba 2015, optax/_src/transform.py scale_by_adam)
plus blackjax/adaptation/mass_matrix.py:364-444 (the diagonal Welford fold, one row at a time) and
blackjax/adaptation/metric_buffers.py:396-450 (cgl_update_batch, oracle/adaptation.py).
"""
from dataclasses import dataclass
from typing import NamedTuple

import numpy as np

from . import prng
from .adaptation import DAState, cgl_update_batch, da_init, moment_block_init, welford_init, welford_update
from .adjusted_mclmc import halton_sequence as halton
from .hmc import F, hmc_kernel, init as hmc_init

OPTIMAL_TARGET_ACCEPTANCE_RATE = 0.651
LOG_UPDATE_CLIP = F(0.35)
EPS_FLOAT = F(1e-20)
LENGTH_FLOOR_FACTOR = F(np.pi / 2)
RECOMPUTE_INTERVAL = 32
POWER_ITERATIONS = 5
FINAL_POWER_ITERATIONS = 20
LAMBDA_EPS = F(1e-6)


def da_update_grad(s, gradient, t0=10, gamma=0.05, kappa=0.75):
    """dual_averaging.py:101-123 with the gradient given directly."""
    log_step, avg_log_step, step, avg_error, mu = s
    reg_step = F(step + t0)
    eta_t = F(F(step) ** F(-kappa))
    avg_error = F((F(1.0) - (F(1.0) / reg_step)) * avg_error + F(gradient) / reg_step)
    log_x = F(mu - (np.sqrt(F(step)) / F(gamma)) * avg_error)
    log_x_avg = F(eta_t * log_step + (F(1.0) - eta_t) * avg_log_step)
    return DAState(log_x, log_x_avg, step + 1, avg_error, mu)


class Adam(NamedTuple):
    count: int
    mu: np.float32
    nu: np.float32


def adam_update(g, s, lr, b1=0.9, b2=0.999, eps=1e-8):
    """optax.adam on a scalar parameter: returns (update, new state); update = -lr * m_hat / (sqrt(v_hat) + eps)."""
    g = F(g)
    mu = F(F(b1) * s.mu + (F(1.0) - F(b1)) * g)
    nu = F(F(b2) * s.nu + (F(1.0) - F(b2)) * g * g)
    count = s.count + 1
    with np.errstate(divide="ignore", invalid="ignore"):
        mu_hat = F(mu / (F(1.0) - F(F(b1) ** F(count))))
        nu_hat = F(nu / (F(1.0) - F(F(b2) ** F(count))))
        upd = F(F(-lr) * (mu_hat / (np.sqrt(nu_hat) + F(eps))))
    return upd, Adam(count, mu, nu)


class ChEESState(NamedTuple):
    step_size: np.float32
    log_step_size_ma: np.float32
    trajectory_length: np.float32
    log_trajectory_length_ma: np.float32
    da: DAState
    optim: Adam
    random_generator_arg: int
    step: int


def chees_init(step_size):
    """chees_adaptation.py:513-523."""
    x = F(step_size)
    return ChEESState(x, F(0.0), x, F(0.0), da_init(x), Adam(0, F(0.0), F(0.0)), 0, 1)


def jitter(i, jitter_amount, max_bits):
    return F(halton(i, max_bits) * F(jitter_amount) + (F(1.0) - F(jitter_amount)))


# ---- the diagonal metric (:61-90) and the Welford fold of its window (:816-824) ---------------------------------------
def welford_fold(w, batch):
    """_fold_welford_batch (:816-824): the single-sample update applied to every row in order."""
    for x in np.asarray(batch, F):
        w = welford_update(w, x)
    return w


def engagement_threshold(D):
    return max(64, int(2 * np.sqrt(D)))


def diagonal_imm(w, threshold, D):
    if w.n >= threshold:
        return np.maximum((w.m2 / F(w.n - 1)).astype(F), EPS_FLOAT).astype(F)
    return np.ones(D, F)


# ---- slow-direction eigenvalue and the floor (:130-236) -------------------------------------------------------------
class EigState(NamedTuple):
    eigenvector: np.ndarray
    lambda_max: np.float32


def eig_state_init(D):
    return EigState((np.ones(D, F) / np.sqrt(F(D))).astype(F), F(1.0))


def power_iteration(matrix, v0, num_iterations):
    matrix = np.asarray(matrix, F)
    v = np.asarray(v0, F)
    for _ in range(num_iterations):
        u = (matrix @ v).astype(F)
        norm = F(np.linalg.norm(u))
        v = (u / (norm if norm > 0 else F(1.0))).astype(F)
    return F(np.dot(v, (matrix @ v).astype(F))), v


def whitened_covariance(block, imm):
    cov = (block.m2 / max(F(block.count - 1), F(1.0))).astype(F)
    s = (F(1.0) / np.sqrt(np.asarray(imm, F))).astype(F)
    return (cov * s[:, None] * s[None, :]).astype(F)


def recompute_eig(block, imm, eig, num_iterations=POWER_ITERATIONS):
    lam, v = power_iteration(whitened_covariance(block, imm), eig.eigenvector, num_iterations)
    return EigState(v, F(max(lam, LAMBDA_EPS)))


def apply_length_floor(trajectory_length, lambda_max, engaged, enable, max_leapfrog_steps, step_size):
    """(consumed length, floor_clipped_by_cap)."""
    if not enable:
        return F(trajectory_length), False
    floor_value = F(LENGTH_FLOOR_FACTOR * np.sqrt(F(lambda_max))) if engaged else F(0.0)
    cap = F(F(max_leapfrog_steps) * F(step_size))
    consumed = F(min(max(F(trajectory_length), floor_value), cap))
    return consumed, bool(engaged and floor_value > cap)


def chees_update(s, prop_q, prop_p, init_q, acc, is_div, *, imm=None, whiten=True, lr, b1=0.9, b2=0.999,
                 target=OPTIMAL_TARGET_ACCEPTANCE_RATE, decay_rate=0.5, max_leapfrog_steps=1000, jitter_amount=1.0, max_bits=10):
    """compute_parameters (chees_adaptation.py:307-511).  With ``whiten`` the criterion is measured in the geometry of the
    inverse mass matrix ``imm`` (:449-466); ``imm=None`` stands for ones, whose whitening is a no-op and is skipped."""
    acc = np.asarray(acc, F)
    nd = ~np.asarray(is_div, bool)
    with np.errstate(divide="ignore", invalid="ignore"):
        hm = F(1.0) / (np.sum(np.where(nd, F(1.0) / acc, F(0.0)), dtype=F) / F(nd.sum()))
    hm = hm if np.isfinite(hm) else F(0.0)
    da_ = da_update_grad(s.da, F(target) - hm)
    eps_ = np.exp(da_.log_step_size).astype(F)
    if np.isfinite(eps_):
        new_eps, new_da, new_log_eps = eps_, da_, da_.log_step_size
    else:
        new_eps, new_da, new_log_eps = s.step_size, s.da, s.da.log_step_size
    uw = F(F(s.step) ** F(-decay_rate))
    new_log_eps_ma = F((F(1.0) - uw) * s.log_step_size_ma + uw * new_log_eps)
    # weighted_empirical_mean :239-247 and nanmean
    w = np.where(nd, acc, F(0.0)).astype(F)
    fin = np.isfinite(prop_q)
    xs = np.where(fin, prop_q, F(0.0)).astype(F)
    w_ = np.where(fin.all(axis=-1), w, F(0.0)).astype(F)
    pmean = (np.sum(w_[:, None] * xs, axis=0, dtype=F) / (np.sum(w_, dtype=F) + EPS_FLOAT)).astype(F)
    imean = np.nanmean(init_q, axis=0, dtype=F).astype(F)
    pc = (prop_q - pmean).astype(F)
    ic = (init_q - imean).astype(F)
    mom = prop_p
    if whiten and imm is not None:
        imm = np.asarray(imm, F)
        inv_sqrt = (F(1.0) / np.sqrt(imm)).astype(F)
        pc = (pc * inv_sqrt).astype(F)
        ic = (ic * inv_sqrt).astype(F)
        mom = ((np.asarray(prop_p, F) * imm).astype(F) * inv_sqrt).astype(F)
    dots = ((np.sum(pc * pc, axis=1, dtype=F) - np.sum(ic * ic, axis=1, dtype=F)) * np.sum(pc * mom, axis=1, dtype=F)).astype(F)
    tg = (jitter(s.random_generator_arg, jitter_amount, max_bits) * s.trajectory_length * dots).astype(F)
    with np.errstate(invalid="ignore"):
        grad = F(np.sum(np.where(nd, acc * tg, F(0.0)), dtype=F) / np.sum(np.where(nd, acc + EPS_FLOAT, F(0.0)), dtype=F))
    log_T = np.log(s.trajectory_length).astype(F)
    upd, optim_ = adam_update(grad, s.optim, lr, b1, b2)
    upd = F(np.clip(upd, -LOG_UPDATE_CLIP, LOG_UPDATE_CLIP))
    log_T_ = F(log_T + upd)
    if np.isfinite(log_T_):
        new_log_T, new_optim = log_T_, optim_
    else:
        new_log_T, new_optim = log_T, s.optim
    new_log_T_ma = F((F(1.0) - uw) * s.log_trajectory_length_ma + uw * new_log_T)
    new_T = np.exp(new_log_T_ma).astype(F)
    new_T = F(np.clip(new_T, new_eps, F(max_leapfrog_steps) * new_eps))
    return ChEESState(new_eps, new_log_eps_ma, new_T, new_log_T_ma, new_da, new_optim, s.random_generator_arg + 1, s.step + 1)


def integration_steps(i, num_leapfrog_steps, jitter_amount, max_bits):
    """integration_steps_fn :775-779."""
    return int(np.ceil(F(jitter(i, jitter_amount, max_bits) * F(num_leapfrog_steps))))


@dataclass(frozen=True)
class ChEESRun:
    """Result of chees_run.  It unpacks as (last HMCState, step_size, num_leapfrog_steps, final ChEESState), the result
    of the identity-metric run; the diagonal metric's results are read by name."""
    state: object
    step_size: np.float32
    num_leapfrog_steps: np.float32
    adaptation_state: ChEESState
    inverse_mass_matrix: np.ndarray
    lambda_max: np.float32
    floor_clipped_by_cap: bool

    def __iter__(self):
        return iter((self.state, self.step_size, self.num_leapfrog_steps, self.adaptation_state))


def chees_run(target, rng_key, positions, step_size, *, lr, b1=0.9, b2=0.999, num_steps=1000, max_sampling_steps=1000,
              target_acceptance_rate=OPTIMAL_TARGET_ACCEPTANCE_RATE, decay_rate=0.5, max_leapfrog_steps=1000,
              jitter_amount=1.0, mass_matrix_estimation=None, window_fraction=0.5, length_floor=True, whiten=True, trace=None):
    """chees_adaptation(...).run.  ``trace`` (list) receives (ChEESState, L, lambda_max, engaged) after every step, the
    last two being the values the next transition uses."""
    if mass_matrix_estimation not in (None, "diagonal"):
        raise ValueError(f"mass_matrix_estimation must be None or 'diagonal', got {mass_matrix_estimation!r}.")
    if not 0.0 <= window_fraction <= 1.0:
        raise ValueError(f"mass_matrix_window_fraction must be in [0.0, 1.0], got {window_fraction}.")
    estimate = mass_matrix_estimation == "diagonal"
    floor_on = estimate and length_floor
    positions = np.asarray(positions, F)
    C, D = positions.shape
    max_bits = int(np.ceil(np.log2(num_steps + max_sampling_steps)))
    window_start = int(window_fraction * num_steps) if estimate else num_steps
    thresh = engagement_threshold(D)
    wf, cov, eig = welford_init(D), moment_block_init(D), eig_state_init(D)
    state = hmc_init(positions, target)
    s = chees_init(step_size)
    keys_step = prng.split(np.asarray(rng_key, np.uint32), num_steps)
    for t in range(num_steps):
        imm = diagonal_imm(wf, thresh, D) if estimate else np.ones(D, F)
        length = s.trajectory_length
        if floor_on:
            length, _ = apply_length_floor(s.trajectory_length, eig.lambda_max, wf.n >= thresh, True, max_leapfrog_steps,
                                           s.step_size)
        L = integration_steps(s.random_generator_arg, F(length / s.step_size), jitter_amount, max_bits)
        keys = prng.split(keys_step[t], C)
        init_q = state.position
        state, info = hmc_kernel(keys, state, target, s.step_size, imm, L)
        s = chees_update(s, info.proposal[0], info.proposal[1], init_q, info.acceptance_rate, info.is_divergent,
                         imm=imm if estimate else None, whiten=whiten, lr=lr, b1=b1, b2=b2, target=target_acceptance_rate,
                         decay_rate=decay_rate, max_leapfrog_steps=max_leapfrog_steps, jitter_amount=jitter_amount,
                         max_bits=max_bits)
        if t >= window_start:
            wf = welford_fold(wf, state.position)
            if floor_on:
                cov = cgl_update_batch(cov, state.position)
                if t % RECOMPUTE_INTERVAL == 0:
                    eig = recompute_eig(cov, imm, eig)
        if trace is not None:
            trace.append((s, L, eig.lambda_max, estimate and wf.n >= thresh))
    eps = np.exp(s.log_step_size_ma).astype(F)
    final_imm = diagonal_imm(wf, thresh, D) if estimate else np.ones(D, F)
    clipped = False
    if floor_on:
        eig = recompute_eig(cov, final_imm, eig, FINAL_POWER_ITERATIONS)
        T_ma = np.exp(s.log_trajectory_length_ma).astype(F)
        consumed, clipped = apply_length_floor(T_ma, eig.lambda_max, wf.n >= thresh, True, max_leapfrog_steps, eps)
        n_lf = F(consumed / eps)
    else:
        n_lf = np.exp(F(s.log_trajectory_length_ma - s.log_step_size_ma)).astype(F)
    return ChEESRun(state, eps, n_lf, s, final_imm, eig.lambda_max, clipped)
