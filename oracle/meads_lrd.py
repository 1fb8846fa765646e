"""Restatement of BlackJAX's MEADS-LRD statistics (``meads_adaptation(..., low_rank_rank=k)``): the shared low-rank
momentum metric of one warm-up step, and the fold parameters computed under it.

TEST INFRASTRUCTURE, float32, built on oracle/meads.py (left unchanged) and the moment block of oracle/adaptation.py.

Follows blackjax/adaptation/meads_adaptation.py and metric_estimators.py:
* accumulated metric         metric_estimators.py:543-615   cov = m2 / max(count - 1, 1), sigma = sqrt(max(diag, 0)) with
                                                            0 -> 1, R = cov / (sigma sigma^T), eigh, top k by |lam - 1|
* top-k order                metric_estimators.py:292-303   argsort(scores)[::-1]
* diagonal fallback          :263-289                       std of all positions (0 -> 1), eye(D, k), ones(k)
* floor                      :292-313                       maximum(lam, 1e-6), NaN kept
* gate                       :549-568                       in window and count >= 2 D, after this step's fold
* damping transform          :215-239, :599-634             (x + ((x U)(lam^-1/2 - 1)) U^T) / sigma, then centred per fold
* step sizes                 :572-597                       the per-fold diagonal heuristic, unchanged
* final metric               :746-771                       the last accumulator if count >= 2 D, else the fallback
"""
import numpy as np

from . import meads as omeads
from .adaptation import MomentBlock, cgl_update_batch, moment_block_init  # noqa: F401  (re-exported)
from .hmc import F

LAM_FLOOR = F(1e-6)


def select_top(lam_all, V, k):
    """select_top_eigenvalues_by_informativeness(tail_handling="raw")."""
    scores = np.abs(lam_all - F(1.0))
    order = np.argsort(scores, kind="stable")[::-1][:k]
    return V[:, order], lam_all[order]


def correlation(m2, count):
    """(sigma, R) of sample_covariance_eigh_low_rank."""
    cov = (np.asarray(m2, F) / F(max(float(count) - 1.0, 1.0))).astype(F)
    sigma = np.sqrt(np.maximum(np.diag(cov), F(0.0))).astype(F)
    sigma = np.where(sigma <= 0, F(1.0), sigma).astype(F)
    inv = (F(1.0) / sigma).astype(F)
    return sigma, (cov * inv[:, None] * inv[None, :]).astype(F)


def from_accumulated(m2, count, k):
    sigma, R = correlation(m2, count)
    lam_all, V = np.linalg.eigh(R)
    U, lam = select_top(lam_all.astype(F), V.astype(F), k)
    return sigma, U, lam


def fallback(positions, k):
    positions = np.asarray(positions, F)
    sigma = positions.std(axis=0, dtype=F).astype(F)
    sigma = np.where(sigma <= 0, F(1.0), sigma).astype(F)
    return sigma, np.eye(positions.shape[1], k, dtype=F), np.ones(k, F)


def floor(lam):
    return np.maximum(np.asarray(lam, F), LAM_FLOOR)


def engaged(acc, in_window, D):
    return bool(in_window) and float(acc.count) >= 2 * D


def step_metric(acc, positions, k, in_window):
    """One step's metric (:549-568): (new accumulator, engaged, sigma, U, lam)."""
    D = positions.shape[1]
    if in_window:
        acc = cgl_update_batch(acc, positions)
    on = engaged(acc, in_window, D)
    sigma, U, lam = from_accumulated(acc.m2, acc.count, k) if on else fallback(positions, k)
    return acc, on, sigma, U, floor(lam)


def final_metric(acc, positions, k):
    D = positions.shape[1]
    sigma, U, lam = from_accumulated(acc.m2, acc.count, k) if float(acc.count) >= 2 * D else fallback(positions, k)
    return sigma, U, floor(lam)


def precondition(x, sigma, U, lam):
    """_low_rank_precondition_pos: M^{1/2}-style whitening of rows x."""
    x = np.asarray(x, F)
    coef = (F(1.0) / np.sqrt(lam) - F(1.0)).astype(F)
    return ((x + ((x @ U).astype(F) * coef) @ U.T) / sigma).astype(F)


def fold_parameters(position, grad, t, num_folds, sigma, U, lam, step_size_multiplier=0.5, damping_slowdown=1.0):
    """The statistics half of one_step with the low-rank metric: (step_size_rolled, scales_rolled, alphas, deltas)."""
    C, D = position.shape
    n = C // num_folds
    eps_r, scales_r, _, _ = omeads.fold_parameters(position, grad, t, num_folds, step_size_multiplier, damping_slowdown)
    alphas = np.zeros(num_folds, F)
    for f in range(num_folds):
        pk = precondition(position[f * n:(f + 1) * n], sigma, U, lam)
        pk = (pk - pk.mean(axis=0, dtype=F)).astype(F)
        gamma = F(max(F(1.0) / np.sqrt(omeads.maximum_eigenvalue(pk)), F(damping_slowdown) / F(F(t + 1) * eps_r[f])))
        alphas[f] = F(F(1.0) - np.exp(F(-2.0) * eps_r[f] * gamma))
    return eps_r, scales_r, alphas, (alphas / F(2.0)).astype(F)


def dense_inverse_mass(sigma, U, lam):
    """M^-1 = diag(sigma) (I + U (diag(lam) - I) U^T) diag(sigma), float64."""
    sigma, U, lam = (np.asarray(a, np.float64) for a in (sigma, U, lam))
    core = np.eye(len(sigma)) + (U * (lam - 1.0)) @ U.T
    return sigma[:, None] * core * sigma[None, :]
