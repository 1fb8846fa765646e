"""Restatement of BlackJAX's generalized HMC kernel (persistent momentum, non-reversible slice acceptance).

TEST INFRASTRUCTURE (see oracle/__init__.py).  float32, every chain of a batch at once.

Follows
* blackjax/mcmc/ghmc.py:30-62     GHMCState, init (momentum ~ N(0, I), slice ~ U(-1, 1))
* blackjax/mcmc/ghmc.py:64-84     momentum_inverse_scale: the 1-D form is an inverse SCALE, squared into M^-1
* blackjax/mcmc/ghmc.py:118-189   kernel: key split, partial momentum refresh, slice translation, ONE velocity-Verlet
                                  step, flip, non-reversible slice accept, flip again
* blackjax/mcmc/ghmc.py:192-213   update_momentum
* blackjax/mcmc/proposal.py:243-264 nonreversible_slice_sampling
* blackjax/mcmc/hmc.py:153-176    the proposal generator (energies, divergence, HMCInfo)
``noise_fn`` (ghmc.py:90,172): a callable on the per-chain noise keys ``split(rng_key)[1]`` returning float32 [C]; default 0.
"""
from typing import NamedTuple

import numpy as np

from . import prng
from .hmc import F, HMCInfo, Metric, integrator_step, safe_energy_diff


class GHMCState(NamedTuple):
    position: np.ndarray
    momentum: np.ndarray
    logdensity: np.ndarray
    logdensity_grad: np.ndarray
    slice: np.ndarray


class PerChainScale(Metric):
    """default_metric(scale ** 2) with one scale vector per chain (scale [C, D]); ghmc.py:83-84."""

    def __init__(self, scale):
        s = np.asarray(scale, F)
        self.imm = (s * s).astype(F)
        self.dense = False
        self.mass_sqrt = (F(1.0) / np.sqrt(self.imm)).astype(F)   # metrics.py:699-704

    def chain(self, c):
        return Metric(self.imm[c])


def init(position, target, keys):
    """ghmc.py:50-62.  keys uint32 [C, 2]."""
    q = np.asarray(position, F)
    logp, g = target(q)
    ks = prng.split(keys, 2)
    momentum = prng.normal(ks[:, 0], (q.shape[1],))            # util.py:89-91 with mu = 0, sigma = 1
    sl = prng.uniform(ks[:, 1], minval=-1.0, maxval=1.0)
    return GHMCState(q, momentum, logp, g, sl)


def _remainder2(x):
    """jnp.remainder(x, 2) for float32: C fmod, then the sign fix-up."""
    r = np.fmod(x, F(2.0)).astype(F)
    return np.where((r != 0) & (r < 0), r + F(2.0), r).astype(F)


def ghmc_kernel(keys, state, target, step_size, momentum_inverse_scale, alpha, delta, divergence_threshold=1000.0,
                margins=None, noise_fn=None):
    """One GHMC transition for every chain.  step_size, alpha, delta: scalars or [C]; momentum_inverse_scale: [D], [C, D]
    (inverse scale, squared here) or a ready ``Metric``.  ``margins`` (test aid, a list): receives |log|slice| - delta_energy|
    per chain, the distance of the accept decision from a tie."""
    if isinstance(momentum_inverse_scale, Metric):
        metric = momentum_inverse_scale
    else:
        s = np.asarray(momentum_inverse_scale, F)
        metric = PerChainScale(s) if s.ndim == 2 else Metric((s * s).astype(F))
    q0, p_prev, logp0, g0, sl = state
    C, D = q0.shape
    alpha = np.broadcast_to(np.asarray(alpha, F), (C,))
    delta = np.broadcast_to(np.asarray(delta, F), (C,))
    eps = np.broadcast_to(np.asarray(step_size, F), (C,))[:, None]
    ks = prng.split(keys, 2)                                         # ghmc.py:169: key_momentum, key_noise
    noise = F(0.0) if noise_fn is None else np.asarray(noise_fn(ks[:, 1]), F)
    fresh = metric.sample_momentum(ks[:, 0], D)
    p0 = (p_prev * np.sqrt(F(1.0) - alpha)[:, None] + np.sqrt(alpha)[:, None] * fresh).astype(F)   # ghmc.py:205-211
    sl = (_remainder2(((sl + F(1.0)) + delta) + noise) - F(1.0)).astype(F)                        # ghmc.py:172
    q1, p1, logp1, g1 = integrator_step(target, metric, q0, p0, g0, eps)
    p1 = (F(-1.0) * p1).astype(F)                                    # hmc.py:158
    e0 = (-logp0 + metric.kinetic_energy(p0)).astype(F)
    e1 = (-logp1 + metric.kinetic_energy(p1)).astype(F)
    d = safe_energy_diff(e0, e1)
    is_div = (-d) > F(divergence_threshold)
    with np.errstate(over="ignore", divide="ignore", invalid="ignore"):
        p_acc = np.minimum(np.exp(d).astype(F), F(1.0))              # proposal.py:253
        acc = np.log(np.abs(sl)).astype(F) <= d                      # proposal.py:254
        af = acc.astype(F)
        if margins is not None:
            margins.append(np.abs(np.log(np.abs(sl)).astype(np.float64) - d.astype(np.float64)))
        sl_next = (sl * (np.exp(-d).astype(F) * af + (F(1.0) - af))).astype(F)   # proposal.py:255
    a = acc[:, None]
    # the sampled state's momentum is flipped once more (ghmc.py:178): accepted -> +p1 of the integrator, rejected -> -p0
    mom = (F(-1.0) * np.where(a, p1, p0)).astype(F)
    new = GHMCState(np.where(a, q1, q0).astype(F), mom, np.where(acc, logp1, logp0).astype(F), np.where(a, g1, g0).astype(F),
                    sl_next)
    info = HMCInfo(p0, p_acc, acc, is_div, e1, (q1, p1, logp1, g1), 1)
    return new, info
