"""Restatement of BlackJAX's Stan-style window adaptation (dual averaging + Welford).

TEST INFRASTRUCTURE (see oracle/__init__.py).  float32.

Follows:
* dual averaging   blackjax/optimizers/dual_averaging.py:87-129, adaptation/step_size.py:65-150
* Welford / IMM    blackjax/adaptation/mass_matrix.py:364-444 (welford), :335-357 (regularised final)
* CGL merge        blackjax/adaptation/metric_buffers.py:334-393 (cgl_merge_two), :396-450 (cgl_update_batch)
* schedule         blackjax/adaptation/staged_adaptation.py:315-405 (build_schedule)
* engine           blackjax/adaptation/staged_adaptation.py:111-307 (_make_engine), :731-754 (one_step),
                   :864-874 (single-chain run), :906-966 (multi-chain shared-epsilon run)
"""
from typing import NamedTuple

import numpy as np

from . import prng
from .hmc import F, HMCState, init as hmc_init


def build_schedule(num_steps, initial_buffer_size=75, final_buffer_size=50, first_window_size=25):
    schedule = []
    if num_steps < 20:
        schedule += [(0, False)] * num_steps
    else:
        if initial_buffer_size + first_window_size + final_buffer_size > num_steps:
            initial_buffer_size = int(0.15 * num_steps)
            final_buffer_size = int(0.1 * num_steps)
            first_window_size = num_steps - initial_buffer_size - final_buffer_size
        schedule += [(0, False)] * initial_buffer_size
        final_buffer_start = num_steps - final_buffer_size
        next_window_size = first_window_size
        next_window_start = initial_buffer_size
        while next_window_start < final_buffer_start:
            current_start, current_size = next_window_start, next_window_size
            if 3 * current_size <= final_buffer_start - current_start:
                next_window_size = 2 * current_size
            else:
                current_size = final_buffer_start - current_start
            next_window_start = current_start + current_size
            schedule += [(1, False)] * (next_window_start - 1 - current_start)
            schedule.append((1, True))
        schedule += [(0, False)] * (num_steps - final_buffer_start)
    return schedule


class DAState(NamedTuple):
    log_step_size: np.float32
    log_step_size_avg: np.float32
    step: int
    avg_error: np.float32
    mu: np.float32


def da_init(initial_step_size):
    x = F(initial_step_size)
    return DAState(np.log(x).astype(F), F(0.0), 1, F(0.0), np.log(F(10.0) * x).astype(F))


def da_update(s, acceptance_rate, target=0.8, t0=10, gamma=0.05, kappa=0.75):
    """dual_averaging.py:101-123; the averaged iterate uses the PRE-update log step."""
    log_step, avg_log_step, step, avg_error, mu = s
    gradient = F(target) - F(acceptance_rate)
    reg_step = F(step + t0)
    eta_t = F(F(step) ** F(-kappa))
    avg_error = F((F(1.0) - (F(1.0) / reg_step)) * avg_error + gradient / reg_step)
    log_x = F(mu - (np.sqrt(F(step)) / F(gamma)) * avg_error)
    log_x_avg = F(eta_t * log_step + (F(1.0) - eta_t) * avg_log_step)
    return DAState(log_x, log_x_avg, step + 1, avg_error, mu)


def da_final(s):
    return np.exp(s.log_step_size_avg).astype(F)


class Welford(NamedTuple):
    mean: np.ndarray
    m2: np.ndarray
    n: int


def welford_init(dim, diagonal=True):
    return Welford(np.zeros(dim, F), np.zeros(dim if diagonal else (dim, dim), F), 0)


def welford_update(w, x):
    """mass_matrix.py:411-433 for ONE draw x[D]."""
    mean, m2, n = w
    n = n + 1
    delta = (x - mean).astype(F)
    mean = (mean + delta / F(n)).astype(F)
    upd = (x - mean).astype(F)
    if m2.ndim == 1:
        m2 = (m2 + delta * upd).astype(F)
    else:
        m2 = (m2 + np.outer(upd, delta)).astype(F)
    return Welford(mean, m2, n)


def cgl_merge(a, b):
    """metric_buffers.py:334-393 merge of two (n, mean, M2) blocks."""
    n_ab = a.n + b.n
    if n_ab == 0:
        return Welford(np.zeros_like(a.mean), np.zeros_like(a.m2), 0)
    delta = (b.mean - a.mean).astype(F)
    mean = (a.mean + delta * F(b.n / n_ab)).astype(F)
    c = F(a.n * b.n / n_ab)
    cross = delta * delta * c if a.m2.ndim == 1 else np.outer(delta, delta) * c
    return Welford(mean, (a.m2 + b.m2 + cross).astype(F), n_ab)


# ---- full moment block (metric_buffers.py:396-450) ------------------------------------------------------------------
# The same Chan-Golub-LeVeque merge as cgl_merge, kept apart because the arithmetic differs: cgl_update_batch keeps the
# count as a float32 (rounded once it passes 2^24) and forms its factors in float32, where cgl_merge takes integer counts
# and rounds each factor once.
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


def batch_block(x):
    """(n, mean, M2) of a batch x[n, D] (metric_buffers.py:396-420, diagonal or dense by caller)."""
    mean = np.mean(x, axis=0, dtype=F)
    c = (x - mean).astype(F)
    return mean, c


def welford_final(w):
    """mass_matrix.py:335-357 Stan regularisation; returns new IMM."""
    mean, m2, n = w
    cov = (m2 / F(n - 1)).astype(F)
    denom = F(n + 5)
    if m2.ndim == 1:
        return (F(n) / denom * cov + F(5.0) / denom * F(1e-3)).astype(F)
    return (F(n) / denom * cov + F(5.0) / denom * F(1e-3) * np.eye(m2.shape[0], dtype=F)).astype(F)


def window_adaptation_run(kernel, target, rng_key, position, num_steps, *, is_mass_matrix_diagonal=True,
                          initial_step_size=1.0, target_acceptance_rate=0.8, shared=False,
                          **kernel_kwargs):
    """``window_adaptation(algorithm, logdensity_fn).run(rng_key, position, num_steps)``.

    ``kernel(keys[C,2], state, target, step_size, imm, **kw) -> (state, info)`` is a batched oracle kernel.

    shared=False: every chain adapts its own (eps, IMM) -- what users get by ``jax.vmap(warmup.run)``
    over (rng_key[c], position[c]); rng_key is uint32[C,2].
    shared=True : the reference's multi-chain shared-epsilon path (staged_adaptation.py:906-966): one key,
    ``split(step_key, C)`` per step, ONE DA update on mean(acceptance_rate), chain-pooled Welford.
    Returns (last_state, step_size, imm, history) where history holds per-step step sizes.
    """
    position = np.asarray(position, F)
    C, D = position.shape
    state = hmc_init(position, target)
    schedule = build_schedule(num_steps)
    diag = is_mass_matrix_diagonal
    if shared:
        keys = prng.split(np.asarray(rng_key, np.uint32), num_steps)          # [T,2]
        da = da_init(initial_step_size)
        imm = np.ones(D, F) if diag else np.eye(D, dtype=F)
        wf = welford_init(D, diag)
        eps = F(initial_step_size)
        hist = []
        for t, (stage, window_end) in enumerate(schedule):
            ck = prng.split(keys[t], C)
            state, info = kernel(ck, state, target, eps, imm, **kernel_kwargs)
            if stage == 1:
                x = state.position
                mean_b = np.mean(x, axis=0, dtype=F)
                cb = (x - mean_b).astype(F)
                m2_b = np.sum(cb * cb, axis=0, dtype=F) if diag else (cb.T @ cb).astype(F)
                wf = cgl_merge(wf, Welford(mean_b, m2_b, C))
            da = da_update(da, np.mean(info.acceptance_rate, dtype=F), target_acceptance_rate)
            eps = np.exp(da.log_step_size).astype(F)
            if window_end:
                imm = welford_final(wf)
                wf = welford_init(D, diag)
                da = da_init(da_final(da))
                eps = np.exp(da.log_step_size).astype(F)
            hist.append(eps)
        return state, da_final(da), imm, np.array(hist, F)
    # per-chain adaptation
    keys = prng.split(np.asarray(rng_key, np.uint32), num_steps)              # [C,T,2]
    das = [da_init(initial_step_size) for _ in range(C)]
    imm = np.ones((C, D), F) if diag else np.tile(np.eye(D, dtype=F), (C, 1, 1))
    wfs = [welford_init(D, diag) for _ in range(C)]
    eps = np.full(C, initial_step_size, F)
    hist = []
    for t, (stage, window_end) in enumerate(schedule):
        if diag:
            state, info = kernel(keys[:, t], state, target, eps, _PerChainDiag(imm), **kernel_kwargs)
        else:  # one dense metric per chain: the batched kernel takes ONE metric, so the chains go through it one by one
            parts = [kernel(keys[c:c + 1, t], type(state)(*(a[c:c + 1] for a in state)), target, eps[c], imm[c],
                            **kernel_kwargs) for c in range(C)]
            state = type(state)(*(np.concatenate([p[0][k] for p in parts]) for k in range(len(state))))
            info = _Acc(np.concatenate([p[1].acceptance_rate for p in parts]))
        for c in range(C):
            if stage == 1:
                wfs[c] = welford_update(wfs[c], state.position[c])
            das[c] = da_update(das[c], info.acceptance_rate[c], target_acceptance_rate)
            eps[c] = np.exp(das[c].log_step_size)
            if window_end:
                imm[c] = welford_final(wfs[c])
                wfs[c] = welford_init(D, diag)
                das[c] = da_init(da_final(das[c]))
                eps[c] = np.exp(das[c].log_step_size)
        hist.append(eps.copy())
    final_eps = np.array([da_final(d) for d in das], F)
    return state, final_eps, imm, np.array(hist, F)


class _Acc(NamedTuple):
    acceptance_rate: np.ndarray


from .hmc import Metric as _Metric  # noqa: E402


class _PerChainDiag(_Metric):
    """Diagonal metric with a different inverse mass vector per chain (imm [C, D])."""

    def __init__(self, imm):
        self.imm = np.asarray(imm, F)
        self.dense = False
        self.mass_sqrt = (F(1.0) / np.sqrt(self.imm)).astype(F)

    def chain(self, c):
        return _Metric(self.imm[c])
