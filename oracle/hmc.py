"""Restatement of BlackJAX's Euclidean metric, velocity-Verlet integrator and HMC kernel.

TEST INFRASTRUCTURE (see oracle/__init__.py).  float32, batched over chains [C, D].

Follows:
* metric           blackjax/mcmc/metrics.py:221-346 (gaussian_euclidean), :701-729 (_format_covariance),
                   blackjax/util.py:23-61 (linear_map), :66-91 (generate_gaussian_noise)
* integrator       blackjax/mcmc/integrators.py:62-152 (generalized_two_stage_integrator),
                   :175-245 (euclidean position/momentum updates), :321-369 (coefficient tables)
* HMC transition   blackjax/mcmc/hmc.py:90-92 (init), :95-112 (flip_momentum), :153-176 (generate),
                   :279-312 (kernel); trajectory.py:136-167 (static_integration), :730-750 (hmc_energy);
                   proposal.py:45-48 (safe_energy_diff), :214-235 (static_binomial_sampling)
"""
from typing import NamedTuple

import numpy as np

from . import prng

F = np.float32

VELOCITY_VERLET = (0.5, 1.0, 0.5)                                   # integrators.py:321
_b1 = 0.1931833275037836
MCLACHLAN = (_b1, 0.5, 1 - 2 * _b1, 0.5, _b1)                        # integrators.py:335-340
_b1y, _a1y = 0.11888010966548, 0.29619504261126
YOSHIDA = (_b1y, _a1y, 0.5 - _b1y, 1 - 2 * _a1y, 0.5 - _b1y, _a1y, _b1y)  # integrators.py:351-357
_b1o, _a1o, _b2o, _a2o = 0.08398315262876693, 0.2539785108410595, 0.6822365335719091, -0.03230286765269967
_b3o, _a3o = 0.5 - _b1o - _b2o, 1 - 2 * (_a1o + _a2o)
OMELYAN = (_b1o, _a1o, _b2o, _a2o, _b3o, _a3o, _b3o, _a2o, _b2o, _a1o, _b1o)  # integrators.py:363-369


# XLA:CPU compiles with llvm::FPOpFusion::Fast, so `x + (eps*coef)*grad` lowers to ONE fused multiply-add
# on FMA-capable hosts; the CUDA path contracts the same way.  Emulated here through float64 (the product of
# two float32 is exact in float64; the double rounding differs from a true FMA with probability ~2^-29).
FMA_CONTRACT = True


def axpy(x, a, y):
    """x + a*y in float32, as a fused multiply-add when FMA_CONTRACT."""
    if FMA_CONTRACT:
        with np.errstate(over="ignore", invalid="ignore"):
            return (np.asarray(x, np.float64) + np.asarray(a, np.float64) * np.asarray(y, np.float64)).astype(F)
    return (x + a * y).astype(F)


class Metric:
    """gaussian_euclidean(inverse_mass_matrix): 1-D => diagonal, 2-D => dense."""

    def __init__(self, inverse_mass_matrix):
        imm = np.asarray(inverse_mass_matrix, F)
        self.imm = imm
        if imm.ndim == 1:
            self.dense = False
            # metrics.py:703-708: mass_matrix_sqrt = 1/sqrt(M^-1)
            self.mass_sqrt = (F(1.0) / np.sqrt(imm)).astype(F)
        elif imm.ndim == 2:
            self.dense = True
            # metrics.py:712-715: L = chol(M^-1) lower ; mass_matrix_sqrt = L^-T
            L = np.linalg.cholesky(imm.astype(np.float64))
            self.mass_sqrt = np.linalg.solve(L.T, np.eye(L.shape[0])).astype(F)
        else:
            raise ValueError(
                "The mass matrix has the wrong number of dimensions:"
                f" expected 1 or 2, got {imm.ndim}."
            )

    def chain(self, c):
        """The metric chain ``c`` runs with, for the single-chain code paths (the U-turn checkpoints of
        oracle/nuts.py).  A shared metric is its own view; per-chain metrics return chain c's row."""
        return self

    def velocity(self, p):
        """linear_map(M^-1, p) (util.py:57-61)."""
        if self.dense:
            return (p @ self.imm.T).astype(F)
        return (self.imm * p).astype(F)

    def sample_momentum(self, keys, dim):
        """metrics.py:260-261 -> util.py:89-91: p = mass_matrix_sqrt (.) normal(key,(D,))."""
        z = prng.normal(keys, (dim,))
        if self.dense:
            return (z @ self.mass_sqrt.T).astype(F)
        return (self.mass_sqrt * z).astype(F)

    def kinetic_energy(self, p):
        """metrics.py:263-270: 0.5 * dot(M^-1 p, p)."""
        return (F(0.5) * np.sum(self.velocity(p) * p, axis=-1, dtype=F)).astype(F)

    def is_turning(self, p_left, p_right, p_sum):
        """metrics.py:272-304 generalised U-turn (<=, OR)."""
        rho = p_sum - (p_right + p_left) / F(2.0)
        tl = np.sum(self.velocity(p_left) * rho, axis=-1, dtype=F) <= 0
        tr = np.sum(self.velocity(p_right) * rho, axis=-1, dtype=F) <= 0
        return tl | tr

    def turning_margin(self, p_left, p_right, p_sum):
        """Test aid (not in the reference): how far the two U-turn dot products are from the decision boundary 0,
        relative to the sum of the magnitudes of their terms -- a value near 0 marks a float tie."""
        rho = p_sum - (p_right + p_left) / F(2.0)
        out = np.full(np.shape(p_left)[:-1], np.inf)
        for pe in (p_left, p_right):
            t = (self.velocity(pe) * rho).astype(np.float64)
            out = np.minimum(out, np.abs(t.sum(-1)) / np.maximum(np.abs(t).sum(-1), 1e-300))
        return out


class LowRankMetric(Metric):
    """gaussian_euclidean_low_rank(sigma, U, lam) (metrics.py:349-467): M^-1 = diag(sigma) (I + U (Lambda - I) U^T) diag(sigma)
    with orthonormal U [D, k]; every operation is O(D k) through _low_rank_matvec (metrics.py:131-177)."""

    def __init__(self, sigma, U, lam):
        self.sigma = np.asarray(sigma, F)
        self.U = np.asarray(U, F)
        self.lam = np.asarray(lam, F)
        self.inv_sigma = (F(1.0) / self.sigma).astype(F)
        self.inv_sqrt_lam = (F(1.0) / np.sqrt(self.lam)).astype(F)
        self.dense = False

    def _lr(self, y, scales):
        """y + U ((s - 1) * (U^T y)), batched over the leading axis."""
        t = (y @ self.U).astype(F)                                  # U^T y
        return (y + ((scales - F(1.0)) * t) @ self.U.T).astype(F)

    def velocity(self, p):
        """kinetic-energy gradient M^-1 p = sigma * lowrank(sigma * p, lam) (metrics.py:430-432)."""
        return (self.sigma * self._lr((self.sigma * p).astype(F), self.lam)).astype(F)

    def sample_momentum(self, keys, dim):
        """metrics.py:389-399: p = (1/sigma) * lowrank(eps, 1/sqrt(lam))."""
        z = prng.normal(keys, (dim,))
        return (self.inv_sigma * self._lr(z, self.inv_sqrt_lam)).astype(F)

    def kinetic_energy(self, p):
        """metrics.py:401-408: 0.5 * dot(q, lowrank(q, lam)), q = sigma * p."""
        q = (self.sigma * p).astype(F)
        return (F(0.5) * np.sum(q * self._lr(q, self.lam), axis=-1, dtype=F)).astype(F)


def integrator_step(target, metric, q, p, g, eps, coefficients=VELOCITY_VERLET):
    """One palindromic two-stage step; eps is f32 scalar or [C,1] (signed)."""
    eps = np.asarray(eps, F)
    logp = None
    v = None
    for i, coef in enumerate(coefficients[:-1]):
        if i % 2 == 0:
            p = axpy(p, eps * F(coef), g)                    # integrators.py:235-239
            v = metric.velocity(p)                            # :242 grad of kinetic energy
        else:
            q = axpy(q, eps * F(coef), v)                    # :199-203
            logp, g = target(q)                               # :204
    p = axpy(p, eps * F(coefficients[-1]), g)                # :134-141 last call
    return q, p, logp, g


def static_integration(target, metric, q, p, logp, g, eps, num_steps, coefficients=VELOCITY_VERLET):
    """trajectory.py:155-165 fori_loop of num_steps integrator steps."""
    for _ in range(int(num_steps)):
        q, p, logp, g = integrator_step(target, metric, q, p, g, eps, coefficients)
    return q, p, logp, g


class HMCState(NamedTuple):
    position: np.ndarray
    logdensity: np.ndarray
    logdensity_grad: np.ndarray


class HMCInfo(NamedTuple):
    momentum: np.ndarray
    acceptance_rate: np.ndarray
    is_accepted: np.ndarray
    is_divergent: np.ndarray
    energy: np.ndarray
    proposal: tuple
    num_integration_steps: int


def init(position, target):
    logp, g = target(np.asarray(position, F))
    return HMCState(np.asarray(position, F), logp, g)


def safe_energy_diff(e0, e1):
    with np.errstate(invalid="ignore"):
        d = (e0 - e1).astype(F)
    return np.where(np.isnan(d), F(-np.inf), d).astype(F)


def hmc_kernel(keys, state, target, step_size, inverse_mass_matrix, num_integration_steps,
               divergence_threshold=1000.0, coefficients=VELOCITY_VERLET):
    """One HMC transition for every chain.  keys: uint32[C,2] (per-chain rng_key)."""
    metric = inverse_mass_matrix if isinstance(inverse_mass_matrix, Metric) else Metric(inverse_mass_matrix)
    q0, logp0, g0 = state
    C, D = q0.shape
    ks = prng.split(keys, 2)                                         # hmc.py:299
    key_momentum, key_integrator = ks[:, 0], ks[:, 1]
    p0 = metric.sample_momentum(key_momentum, D)                      # hmc.py:302
    eps = np.asarray(step_size, F)
    if eps.ndim == 1:
        eps = eps[:, None]
    q1, p1, logp1, g1 = static_integration(target, metric, q0, p0, logp0, g0, eps,
                                           num_integration_steps, coefficients)
    p1 = (F(-1.0) * p1).astype(F)                                    # flip_momentum hmc.py:158
    e0 = (-logp0 + metric.kinetic_energy(p0)).astype(F)              # hmc.py:159
    e1 = (-logp1 + metric.kinetic_energy(p1)).astype(F)              # hmc.py:160
    delta = safe_energy_diff(e0, e1)                                 # hmc.py:161
    is_div = (-delta) > F(divergence_threshold)                      # hmc.py:162
    with np.errstate(over="ignore"):
        p_acc = np.minimum(np.exp(delta).astype(F), F(1.0))          # proposal.py:225
    u = prng.uniform(key_integrator)                                  # proposal.py:226 (same key)
    acc = u < p_acc
    a = acc[:, None]
    new = HMCState(np.where(a, q1, q0).astype(F), np.where(acc, logp1, logp0).astype(F),
                   np.where(a, g1, g0).astype(F))
    info = HMCInfo(p0, p_acc, acc, is_div, e1, (q1, p1, logp1, g1), int(num_integration_steps))
    return new, info


def dynamic_hmc_kernel(keys, state, random_generator_arg, target, step_size, inverse_mass_matrix,
                       divergence_threshold=1000.0, coefficients=VELOCITY_VERLET, multinomial=False):
    """Dynamic HMC (blackjax/mcmc/dynamic_hmc.py:97-128) with the default ``integration_steps_fn =
    randint(key, (), 1, 10)`` (:66) and ``next_random_arg_fn = split(key)[1]`` (:65): every chain draws its own number
    of integration steps from its ``random_generator_arg`` and runs the static HMC kernel with it.  Restated chain by
    chain (the step counts differ).  Returns (new_state, info, next_random_generator_arg, steps)."""
    q0, logp0, g0 = state
    C = q0.shape[0]
    steps = prng.randint(random_generator_arg, (), 1, 10)                       # :109-111
    base = mhmc_kernel if multinomial else hmc_kernel
    eps = np.asarray(step_size, F)
    news, infos = [], []
    for c in range(C):
        st = (q0[c:c + 1], logp0[c:c + 1], g0[c:c + 1])
        new, info = base(keys[c:c + 1], st, target, eps[c:c + 1] if eps.ndim == 1 else eps, inverse_mass_matrix,
                         int(steps[c]), divergence_threshold, coefficients)   # :113-120
        news.append(new)
        infos.append(info)
    new = HMCState(*[np.concatenate([n[i] for n in news]) for i in range(3)])
    nxt = prng.split(random_generator_arg, 2)[:, 1]                             # :121
    return new, infos, nxt, steps


def mhmc_kernel(keys, state, target, step_size, inverse_mass_matrix, num_integration_steps,
                divergence_threshold=1000.0, coefficients=VELOCITY_VERLET):
    """Multinomial HMC transition (hmc.py:181-248 multinomial_hmc_proposal + trajectory.py:170-232
    static_progressive_integration + proposal.py:118-143 progressive_uniform_sampling) for every chain."""
    from .nuts import expit, logaddexp
    metric = inverse_mass_matrix if isinstance(inverse_mass_matrix, Metric) else Metric(inverse_mass_matrix)
    q0, logp0, g0 = state
    C, D = q0.shape
    ks = prng.split(keys, 2)                                         # hmc.py:299
    key_momentum, key_integrator = ks[:, 0], ks[:, 1]
    p0 = metric.sample_momentum(key_momentum, D)
    eps = np.asarray(step_size, F)
    if eps.ndim == 1:
        eps = eps[:, None]
    h0 = (-logp0 + metric.kinetic_energy(p0)).astype(F)              # trajectory.py:211
    prop = dict(q=q0.copy(), p=p0.copy(), g=g0.copy(), logp=logp0.copy(), energy=h0.copy(),
                weight=np.zeros(C, F), slpa=np.full(C, -np.inf, F))  # :212
    q, p, logp, g = q0, p0, logp0, g0
    any_div = np.zeros(C, bool)
    for i in range(int(num_integration_steps)):
        step_key = prng.fold_in(key_integrator, i)                   # :216
        q, p, logp, g = integrator_step(target, metric, q, p, g, eps, coefficients)
        e_new = (-logp + metric.kinetic_energy(p)).astype(F)
        w_new = safe_energy_diff(h0, e_new)                          # proposal.py:94-98
        slpa_new = np.minimum(w_new, F(0.0)).astype(F)
        any_div |= (-w_new) > F(divergence_threshold)                # :220-221
        with np.errstate(invalid="ignore"):
            p_accept = expit(w_new - prop["weight"])                 # proposal.py:122
        acc = prng.uniform(step_key) < p_accept
        a = acc[:, None]
        prop["q"] = np.where(a, q, prop["q"]).astype(F)
        prop["p"] = np.where(a, p, prop["p"]).astype(F)
        prop["g"] = np.where(a, g, prop["g"]).astype(F)
        prop["logp"] = np.where(acc, logp, prop["logp"]).astype(F)
        prop["energy"] = np.where(acc, e_new, prop["energy"]).astype(F)
        prop["weight"] = logaddexp(prop["weight"], w_new)
        prop["slpa"] = logaddexp(prop["slpa"], slpa_new)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        acc_rate = (np.exp(prop["slpa"]).astype(F) / F(num_integration_steps)).astype(F)   # hmc.py:232
    new = HMCState(prop["q"], prop["logp"], prop["g"])
    info = HMCInfo(p0, acc_rate, np.ones(C, bool), any_div, prop["energy"],
                   (prop["q"], prop["p"], prop["logp"], prop["g"]), int(num_integration_steps))
    return new, info
