"""Restatement of BlackJAX's low-rank window adaptation (``window_adaptation_low_rank``, buffer_policy="reset") in
float64 numpy, for the tests of ``blackjax_b200.window_adaptation_low_rank``.

TEST INFRASTRUCTURE.  Follows blackjax/adaptation:
* estimator                metric_estimators.py:618-808   _compute_low_rank_metric on a [B, d] buffer with n valid rows
                                                          (n_safe = max(n, 2); when the window outgrew the buffer all B
                                                          rows are valid but the sums are still divided by n)
* SPD utilities            metric_estimators.py:77-142    _relative_pd_floor, _spd_mean
* reset core               metric_recipes.py:601-700      circular buffer write at idx % B, final + hard reset
* buffer rows              low_rank_adaptation.py:604-605 B = min(2 max(num_steps // 5, 128), num_steps)
* growing schedule         low_rank_adaptation.py:310-450 incl. the is_late rule
* engine loop              staged_adaptation.py:153-307,906-966  pooled: one dual-averaging update on the mean
                                                          acceptance, the stacked rows of all chains in the buffer
The accumulator form (count, mean, M2 per stream, Chan merge) that the device uses is restated next to the row form.
"""
from typing import NamedTuple

import numpy as np

EPS64 = np.finfo(np.float64).eps
TINY64 = np.finfo(np.float64).tiny


# ---- SPD utilities --------------------------------------------------------------------------------------------------
def relative_pd_floor(vals):
    return EPS64 * max(np.max(np.abs(vals)), TINY64)


def spd_mean(A, B):
    """A # B via the eigendecomposition of B (metric_estimators.py:102-142)."""
    vb, Vb = np.linalg.eigh(B)
    vb = np.maximum(vb, relative_pd_floor(vb))
    sb = np.sqrt(vb)
    M = (1.0 / sb)[:, None] * (Vb.T @ A @ Vb) * (1.0 / sb)[None, :]
    vm, Vm = np.linalg.eigh(M)
    vm = np.maximum(vm, relative_pd_floor(vm))
    W = Vb @ (sb[:, None] * Vm)
    return (W * np.sqrt(vm)[None, :]) @ W.T


def _finish(X, A, sigma, mu_star, d, max_rank, gamma, cutoff, Sx=None, Sa=None):
    """Steps 3-9 from the scaled rows X, A (or their scatters Sx = X^T X, Sa = A^T A)."""
    if Sx is None:
        Sx, Sa = X.T @ X, A.T @ A
    # right singular vectors of X = eigenvectors of X^T X, by descending singular value
    wx, Vx = np.linalg.eigh(Sx)
    wa, Va = np.linalg.eigh(Sa)
    Ux = Vx[:, ::-1][:, :max_rank]
    Ua = Va[:, ::-1][:, :max_rank]
    Q, _ = np.linalg.qr(np.concatenate([Ux, Ua], axis=1))
    q = Q.shape[1]
    Cx = Q.T @ Sx @ Q / gamma + np.eye(q)
    Ca = Q.T @ Sa @ Q / gamma + np.eye(q)
    Sigma = spd_mean(Cx, np.linalg.inv(Ca))
    vals, vecs = np.linalg.eigh(Sigma)
    vals = np.maximum(vals, relative_pd_floor(vals))
    U_full = Q @ vecs
    r = min(max_rank, q)
    order = np.argsort(-np.abs(vals - 1.0), kind="stable")[:r]
    U = U_full[:, order]
    lam_raw = vals[order]
    lam = np.where((lam_raw < 1.0 / cutoff) | (lam_raw > cutoff), lam_raw, 1.0)
    if r < max_rank:
        U = np.concatenate([U, np.zeros((d, max_rank - r))], axis=1)
        lam = np.concatenate([lam, np.ones(max_rank - r)])
    return sigma, mu_star, U, lam


def compute_low_rank_metric(draws_buffer, grads_buffer, n, max_rank, gamma, cutoff):
    """_compute_low_rank_metric: (sigma, mu_star, U, lam), float64."""
    X0 = np.asarray(draws_buffer, np.float64)
    G0 = np.asarray(grads_buffer, np.float64)
    B, d = X0.shape
    mask = (np.arange(B) < n).astype(np.float64)
    n_safe = float(max(n, 2))
    mean_x = (mask[:, None] * X0).sum(0) / n_safe
    mean_g = (mask[:, None] * G0).sum(0) / n_safe
    dx = mask[:, None] * (X0 - mean_x)
    dg = mask[:, None] * (G0 - mean_g)
    var_x = (dx ** 2).sum(0) / n_safe
    var_g = (dg ** 2).sum(0) / n_safe
    sigma = np.clip(np.clip(var_x / np.maximum(var_g, 1e-10), 0.0, None) ** 0.25, 1e-20, 1e20)
    mu_star = mean_x + sigma ** 2 * mean_g
    return _finish(dx / sigma, dg * sigma, sigma, mu_star, d, max_rank, gamma, cutoff)


# ---- the accumulator form -------------------------------------------------------------------------------------------
class Moments(NamedTuple):
    count: float
    mean: np.ndarray
    m2: np.ndarray


def moments_init(d):
    return Moments(0.0, np.zeros(d), np.zeros((d, d)))


def moments_fold(m, rows):
    """Chan merge of a batch of rows into (count, mean, M2)."""
    rows = np.asarray(rows, np.float64).reshape(-1, m.mean.shape[0])
    nb = float(rows.shape[0])
    mb = rows.mean(0)
    cb = rows - mb
    m2b = cb.T @ cb
    if m.count == 0.0:
        return Moments(nb, mb, m2b)
    ab = m.count + nb
    delta = mb - m.mean
    return Moments(ab, m.mean + delta * (nb / ab), m.m2 + m2b + np.outer(delta, delta) * (m.count * nb / ab))


def metric_from_moments(mx, mg, n, max_rank, gamma, cutoff):
    """The estimator from the accumulators of the retained rows (count c) and the step count n: x_bar = (c / n) mean,
    scatter M2 + c d d^T with d = mean - x_bar."""
    d = mx.mean.shape[0]
    n_safe = float(max(n, 2))
    c = mx.count
    xbar, gbar = c * mx.mean / n_safe, c * mg.mean / n_safe
    ex, eg = mx.mean - xbar, mg.mean - gbar
    Sx0 = mx.m2 + c * np.outer(ex, ex)
    Sg0 = mg.m2 + c * np.outer(eg, eg)
    var_x, var_g = np.diag(Sx0) / n_safe, np.diag(Sg0) / n_safe
    sigma = np.clip(np.clip(var_x / np.maximum(var_g, 1e-10), 0.0, None) ** 0.25, 1e-20, 1e20)
    mu_star = xbar + sigma ** 2 * gbar
    Sx = Sx0 / np.outer(sigma, sigma)
    Sa = Sg0 * np.outer(sigma, sigma)
    return _finish(None, None, sigma, mu_star, d, max_rank, gamma, cutoff, Sx=Sx, Sa=Sa)


def implied_inverse_mass_matrix(sigma, U, lam):
    """diag(sigma) (I + U (diag(lam) - I) U^T) diag(sigma)"""
    sigma, U, lam = (np.asarray(a, np.float64) for a in (sigma, U, lam))
    inner = np.eye(sigma.shape[0]) + (U * (lam - 1.0)[None, :]) @ U.T
    return sigma[:, None] * inner * sigma[None, :]


# ---- the reset core: circular buffer of B steps (pooled: B x C rows) ------------------------------------------------
def buffer_size(num_steps):
    return min(2 * max(num_steps // 5, 128), max(num_steps, 1))


class ResetCore:
    """metric_recipes.py:601-700 with one buffer slot per step holding the rows of all C chains."""

    def __init__(self, d, max_rank, gamma, cutoff, B, C=1):
        self.d, self.k, self.gamma, self.cutoff, self.B, self.C = d, max_rank, gamma, cutoff, B, C
        self.sigma, self.U, self.lam = np.ones(d), np.zeros((d, max_rank)), np.ones(max_rank)
        self.mu_star = np.zeros(d)
        self._reset()

    def _reset(self):
        self.draws = np.zeros((self.B, self.C, self.d))
        self.grads = np.zeros((self.B, self.C, self.d))
        self.idx = 0

    def update(self, x, g):
        self.draws[self.idx % self.B] = np.asarray(x, np.float64).reshape(self.C, self.d)
        self.grads[self.idx % self.B] = np.asarray(g, np.float64).reshape(self.C, self.d)
        self.idx += 1

    def final(self):
        rows = min(self.idx, self.B)
        X = self.draws[:rows].reshape(-1, self.d)
        G = self.grads[:rows].reshape(-1, self.d)
        self.sigma, self.mu_star, self.U, self.lam = compute_low_rank_metric(X, G, self.C * self.idx, self.k, self.gamma,
                                                                             self.cutoff)
        self._reset()


# ---- schedules ------------------------------------------------------------------------------------------------------
def build_growing_window_schedule(num_steps, early_window=0.3, step_size_window=0.15, early_window_size=10,
                                  window_size=80, window_growth=1.5):
    if num_steps < 20:
        return [(0, False)] * num_steps
    final_buffer_size = max(int(round(step_size_window * num_steps)), 1)
    final_buffer_start = num_steps - final_buffer_size
    early_end = min(max(int(round(early_window * num_steps)), 1), final_buffer_start)
    out, pos = [], 0
    while pos < early_end:
        size = min(early_window_size, early_end - pos)
        out += [(1, False)] * (size - 1) + [(1, True)]
        pos += size
    current = window_size
    while pos < final_buffer_start:
        remaining = final_buffer_start - pos
        next_size = max(current + 1, int(round(current * window_growth)))
        if (pos + current) + next_size > final_buffer_start:
            out += [(1, False)] * (remaining - 1) + [(1, True)]
            pos += remaining
            break
        out += [(1, False)] * (current - 1) + [(1, True)]
        pos += current
        current = next_size
    out += [(0, False)] * (num_steps - pos)
    return out


def window_sizes(schedule):
    ends = [t for t, (_, e) in enumerate(schedule) if e]
    return np.diff(np.concatenate([[-1], ends])).astype(int).tolist()


# ---- dual averaging in float32 (k_shared_adapt's arithmetic) and the pooled engine loop ------------------------------
F = np.float32


# kept apart from adaptation.da_update: its scalar step ** -0.75 and np.power here differ by an ulp at some steps
class DA(NamedTuple):
    log_step: F
    log_avg: F
    step: F
    err: F
    mu: F


def da_init(eps):
    eps = F(eps)
    return DA(np.log(eps), F(0), F(1), F(0), np.log(F(10) * eps))


def da_update(s, accept_mean, target):
    gradient = F(target) - F(accept_mean)
    reg = s.step + F(10)
    eta = np.power(s.step, F(-0.75))
    err = (F(1) - F(1) / reg) * s.err + gradient / reg
    log_x = s.mu - (np.sqrt(s.step) / F(0.05)) * err
    log_avg = eta * s.log_step + (F(1) - eta) * s.log_avg
    return DA(F(log_x), F(log_avg), s.step + F(1), F(err), s.mu)


class PooledRun(NamedTuple):
    step_sizes: list      # float32 step size after every step
    metrics: list         # (t, sigma, mu_star, U, lam) at every window end
    final_step_size: float
    mu_star: np.ndarray


def run_pooled(draws, grads, accept, schedule, max_rank=10, initial_step_size=1.0, target=0.8, gamma=1e-5, cutoff=2.0,
               num_steps=None):
    """The pooled warm-up driven by given per-step draws / gradients [T, C, D] and acceptance rates [T, C]."""
    T, C, d = draws.shape
    num_steps = T if num_steps is None else num_steps
    core = ResetCore(d, max_rank, gamma, cutoff, buffer_size(num_steps), C)
    da = da_init(initial_step_size)
    hist, metrics = [], []
    for t, (stage, end) in enumerate(schedule[:T]):
        if stage == 1:
            core.update(draws[t], grads[t])
        da = da_update(da, np.mean(np.asarray(accept[t], np.float64)), target)
        if end:
            core.final()
            metrics.append((t, core.sigma, core.mu_star, core.U, core.lam))
            da = da_init(np.exp(da.log_avg))
        hist.append(float(np.exp(da.log_step)))
    return PooledRun(hist, metrics, float(np.exp(da.log_avg)), core.mu_star)
