"""MALA (blackjax/mcmc/mala.py:68-117, diffusions.py:32-59, proposal.py:45-48,184-233) restated in float32 NumPy for a
batch of chains, with the decision margin |u - p_accept| per chain."""
import numpy as np

from . import prng

F = np.float32


def transition_energy(x, y, logp_y, g_y, eps):
    """E(x -> y) = -logp_y + (0.25 * (1 / eps)) * sum (x - y - eps g_y)^2   (mala.py:80-92); eps [C, 1]."""
    t = ((x - y).astype(F) - (eps * g_y).astype(F)).astype(F)
    w = (F(0.25) * (F(1.0) / eps[:, 0]).astype(F)).astype(F)
    return (-logp_y + (w * np.sum(t * t, axis=-1, dtype=F)).astype(F)).astype(F)


def step(keys, q, logp, g, logdensity_fn, step_size):
    """One transition of every chain.  keys [C, 2]; step_size scalar or [C].  Returns ((q, logp, g), info) where info
    holds acceptance_rate, is_accepted, the proposal (position, logdensity, grad) and margin = |u - p_accept|."""
    q, logp, g = (np.asarray(a, F) for a in (q, logp, g))
    C, D = q.shape
    eps = np.broadcast_to(np.asarray(step_size, F), (C,)).astype(F)[:, None]
    ks = prng.split(keys)                              # key_integrator, key_rmh  mala.py:104
    xi = prng.normal(ks[:, 0], (D,))
    y = ((q + (eps * g).astype(F)).astype(F) + (np.sqrt((F(2.0) * eps).astype(F)).astype(F) * xi).astype(F)).astype(F)
    logp_y, g_y = logdensity_fn(y)
    logp_y, g_y = np.asarray(logp_y, F), np.asarray(g_y, F)
    with np.errstate(all="ignore"):
        e_new = transition_energy(q, y, logp_y, g_y, eps)
        e_prev = transition_energy(y, q, logp, g, eps)
        la = (e_prev - e_new).astype(F)
        la = np.where(np.isnan(la), F(-np.inf), la)    # safe_energy_diff  proposal.py:45-48
        p = np.minimum(np.exp(la), F(1.0)).astype(F)
    u = prng.uniform(ks[:, 1])
    acc = u < p
    out = (np.where(acc[:, None], y, q), np.where(acc, logp_y, logp), np.where(acc[:, None], g_y, g))
    return out, dict(acceptance_rate=p, is_accepted=acc, proposal=(y, logp_y, g_y), margin=np.abs(u - p))
