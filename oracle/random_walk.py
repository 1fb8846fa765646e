"""Random-walk Metropolis (blackjax/mcmc/random_walk.py:94-109,182-185,453-530, util.py:24-91, proposal.py:184-235)
restated in float32 NumPy for a batch of chains, with the decision inputs per chain.

One transition with the chain key ``key``: ``key_proposal, key_accept = split(key)``; ``z = normal(key_proposal, (D,))``;
``lin = sigma * z`` (scalar or [D] sigma) or ``sigma @ z`` ([D, D]); the candidate ``y = x + lin`` (additive) or
``y = mean + lin`` (independent); ``E(a, b) = -logp(b) - f(b, a)``; ``log_a = safe_energy_diff(E(y, x), E(x, y))``;
``p = min(1, exp(log_a))``; accept when ``uniform(key_accept) < p``.  The stored ``logp(x)`` is used as given.

The device's correction ``f`` (``gaussian_logdensity``) is ``f(b, a) = -0.5 sum ((a - mean) (1 / sigma))^2``; here
``f`` may also be any callable ``f(new, prev)`` of ``(position, logdensity)`` pairs, as the reference's
``proposal_logdensity_fn`` is, and ``propose`` any callable ``(key_proposal, x) -> y`` (the reference's generators)."""
import numpy as np

from . import prng

F = np.float32


def linear_map(sigma, z):
    """util.py linear_map: ``sigma * z`` for a scalar or [D] sigma, ``sigma @ z`` for [D, D] (per chain, float32 out)."""
    sigma = np.asarray(sigma, F)
    if sigma.ndim <= 1:
        return (sigma * z).astype(F)
    return np.einsum("ij,cj->ci", sigma.astype(np.float64), z.astype(np.float64)).astype(F)


def gaussian_logdensity(mean, sigma):
    """The device's ``gaussian_logdensity(mean, sigma)``: f(new, prev) = -0.5 sum ((prev.x - mean) (1 / sigma))^2."""
    mean, inv = np.asarray(mean, F), (F(1.0) / np.asarray(sigma, F)).astype(F)

    def f(new, prev):
        d = ((np.asarray(prev[0], F) - mean).astype(F) * inv).astype(F)
        return (F(-0.5) * np.sum(d * d, axis=-1, dtype=F)).astype(F)

    return f


def propose(keys_proposal, x, sigma, mean=None):
    """The Gaussian candidate: x + lin (mean None) or mean + lin."""
    C, D = x.shape
    lin = linear_map(sigma, prng.normal(keys_proposal, (D,)))
    base = x if mean is None else np.broadcast_to(np.asarray(mean, F), (C, D))
    return (base + lin).astype(F)


def step(keys, x, logp, logdensity_fn, sigma=None, mean=None, proposal_logdensity_fn=None, proposal=None):
    """One transition of every chain.  keys [C, 2]; x [C, D]; logp [C] (used as given); logdensity_fn maps [C, D] to
    (logp [C], anything); the candidate is ``proposal(key_proposal [C, 2], x)`` when given, else :func:`propose` with
    ``sigma`` and ``mean``.  Returns ((x, logp), info) with acceptance_rate, is_accepted, the candidate (y, logp_y),
    log_a and log_u = log(uniform(key_accept))."""
    x = np.asarray(x, F)
    C = x.shape[0]
    logp = np.broadcast_to(np.asarray(logp, F), (C,)).astype(F)
    ks = prng.split(np.asarray(keys, np.uint32))
    y = proposal(ks[:, 0], x) if proposal is not None else propose(ks[:, 0], x, sigma, mean)
    y = np.asarray(y, F)
    logp_y = np.asarray(logdensity_fn(y)[0], F)
    with np.errstate(all="ignore"):
        if proposal_logdensity_fn is None:
            e_prev, e_new = -logp, -logp_y
        else:
            e_prev = (-logp - np.asarray(proposal_logdensity_fn((x, logp), (y, logp_y)), F)).astype(F)
            e_new = (-logp_y - np.asarray(proposal_logdensity_fn((y, logp_y), (x, logp)), F)).astype(F)
        la = (e_prev - e_new).astype(F)
        la = np.where(np.isnan(la), F(-np.inf), la).astype(F)   # safe_energy_diff
        p = np.minimum(np.exp(la), F(1.0)).astype(F)
        u = prng.uniform(ks[:, 1])
        acc = u < p
        log_u = np.log(u)
    out = (np.where(acc[:, None], y, x).astype(F), np.where(acc, logp_y, logp).astype(F))
    return out, dict(acceptance_rate=p, is_accepted=acc, candidate=(y, logp_y), log_a=la, log_u=log_u)
