"""Restatement of BlackJAX's ChEES warm-up with ``mass_matrix_estimation="diagonal"``: the ensemble-estimated diagonal
inverse mass matrix, the whitened ChEES criterion and the slow-direction trajectory-length floor.

TEST INFRASTRUCTURE, float32, built on oracle/chees.py (whose identity-metric functions it leaves as they are).

Follows blackjax/adaptation/chees_adaptation.py:
* engagement threshold      :61-72       max(64, int(2 sqrt(D)))
* engaged-or-ones metric    :75-90       max(m2 / (n - 1), 1e-20) once n >= threshold
* power iteration           :147-166     warm-started, norm guarded to 1 when 0, Rayleigh quotient
* recompute                 :169-189     covariance m2 / max(count - 1, 1), whitened by 1/sqrt(imm) on both sides
* length floor              :192-236     min(max(T, (pi/2) sqrt(lambda_max)), max_leapfrog_steps * eps) when engaged
* whitened criterion        :449-466
* run loop                  :797-1001    window start int(fraction * num_steps), recompute when t % 32 == 0 in window
plus blackjax/adaptation/mass_matrix.py:364-444 (the Welford fold, one row at a time) and
blackjax/adaptation/metric_buffers.py:396-450 (cgl_update_batch).
"""
from typing import NamedTuple

import numpy as np

from oracle import prng
from oracle.chees import (EPS_FLOAT, LOG_UPDATE_CLIP, ChEESState, adam_update, chees_init, da_update_grad,
                          integration_steps, jitter)
from oracle.hmc import F, hmc_kernel, init as hmc_init

LENGTH_FLOOR_FACTOR = F(np.pi / 2)
RECOMPUTE_INTERVAL = 32
POWER_ITERATIONS = 5
FINAL_POWER_ITERATIONS = 20
LAMBDA_EPS = F(1e-6)


# ---- diagonal Welford accumulator (mass_matrix.py:390-444, is_diagonal_matrix=True) --------------------------------
class Welford(NamedTuple):
    mean: np.ndarray
    m2: np.ndarray
    n: int


def welford_init(D):
    return Welford(np.zeros(D, F), np.zeros(D, F), 0)


def welford_fold(w, batch):
    """_fold_welford_batch (:816-824): the single-sample update applied to every row in order."""
    mean, m2, n = w.mean, w.m2, w.n
    for x in np.asarray(batch, F):
        n += 1
        delta = (x - mean).astype(F)
        mean = (mean + delta / F(n)).astype(F)
        m2 = (m2 + delta * (x - mean)).astype(F)
    return Welford(mean, m2, n)


def engagement_threshold(D):
    return max(64, int(2 * np.sqrt(D)))


def diagonal_imm(w, threshold, D):
    if w.n >= threshold:
        return np.maximum((w.m2 / F(w.n - 1)).astype(F), EPS_FLOAT).astype(F)
    return np.ones(D, F)


# ---- full moment block (metric_buffers.py:396-450) ------------------------------------------------------------------
class MomentBlock(NamedTuple):
    count: np.float32
    mean: np.ndarray
    m2: np.ndarray


def moment_block_init(D):
    return MomentBlock(F(0.0), np.zeros(D, F), np.zeros((D, D), F))


def cgl_update_batch(block, batch):
    batch = np.asarray(batch, F)
    n_a, n_b = block.count, F(batch.shape[0])
    mean_b = np.mean(batch, axis=0, dtype=F).astype(F)
    cb = (batch - mean_b).astype(F)
    m2_b = (cb.T @ cb).astype(F)
    n_ab = F(n_a + n_b)
    safe = n_ab if n_ab > 0 else F(1.0)
    delta = (mean_b - block.mean).astype(F)
    mean = (block.mean + delta * F(n_b / safe)).astype(F)
    m2 = (block.m2 + m2_b + np.outer(delta, delta).astype(F) * F(n_a * n_b / safe)).astype(F)
    return MomentBlock(n_ab, mean, m2)


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


# ---- whitened criterion (:307-511 with :449-466) --------------------------------------------------------------------
def chees_update(s, prop_q, prop_p, init_q, acc, is_div, *, imm=None, whiten=True, lr, b1=0.9, b2=0.999, target=0.651,
                 decay_rate=0.5, max_leapfrog_steps=1000, jitter_amount=1.0, max_bits=10):
    """oracle.chees.chees_update with the criterion measured in the geometry of ``imm`` (None: ones)."""
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
    w = np.where(nd, acc, F(0.0)).astype(F)
    fin = np.isfinite(prop_q)
    xs = np.where(fin, prop_q, F(0.0)).astype(F)
    w_ = np.where(fin.all(axis=-1), w, F(0.0)).astype(F)
    pmean = (np.sum(w_[:, None] * xs, axis=0, dtype=F) / (np.sum(w_, dtype=F) + EPS_FLOAT)).astype(F)
    imean = np.nanmean(init_q, axis=0, dtype=F).astype(F)
    pc = (prop_q - pmean).astype(F)
    ic = (init_q - imean).astype(F)
    mm = np.asarray(prop_p, F)
    if whiten:
        imm_ = np.ones(pc.shape[1], F) if imm is None else np.asarray(imm, F)
        inv_sqrt = (F(1.0) / np.sqrt(imm_)).astype(F)
        pc = (pc * inv_sqrt).astype(F)
        ic = (ic * inv_sqrt).astype(F)
        mm = ((mm * imm_).astype(F) * inv_sqrt).astype(F)
    dots = ((np.sum(pc * pc, axis=1, dtype=F) - np.sum(ic * ic, axis=1, dtype=F)) * np.sum(pc * mm, axis=1, dtype=F)).astype(F)
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


# ---- the run loop (:737-1001) ---------------------------------------------------------------------------------------
class MetricRun(NamedTuple):
    state: object
    step_size: np.float32
    num_leapfrog_steps: np.float32
    adaptation_state: ChEESState
    inverse_mass_matrix: np.ndarray
    lambda_max: np.float32
    floor_clipped_by_cap: bool


def chees_run(target, rng_key, positions, step_size, *, lr, b1=0.9, b2=0.999, num_steps=1000, max_sampling_steps=1000,
              target_acceptance_rate=0.651, decay_rate=0.5, max_leapfrog_steps=1000, jitter_amount=1.0,
              mass_matrix_estimation=None, window_fraction=0.5, length_floor=True, whiten=True, trace=None):
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
        s = chees_update(s, info.proposal[0], info.proposal[1], init_q, info.acceptance_rate, info.is_divergent, imm=imm,
                         whiten=whiten if estimate else True, lr=lr, b1=b1, b2=b2, target=target_acceptance_rate,
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
    return MetricRun(state, eps, n_lf, s, final_imm, eig.lambda_max, clipped)
