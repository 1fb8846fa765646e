"""Restatement of BlackJAX's GIST samplers: the seam and its trajectory-length and step-size instances.

TEST INFRASTRUCTURE (see oracle/__init__.py).  float32, batched over chains [C, D]; the rollouts and searches run every
chain in lock step and keep the state of the chains that have stopped.

Follows:
* seam              blackjax/mcmc/composed/_seam.py:143-208 (_step)
* trajectory length blackjax/mcmc/composed/trajectory_length.py:134-206 (num_steps_to_uturn), :295-301
                    (_step_distribution), :304-367 (tuning_parameter_fn, apply_fn; the proposal is re-integrated, which
                    the reference's own tests pin to the cached rollout state)
* step size         blackjax/mcmc/composed/step_size.py:142-291 (step_size_selector), :294-346
"""
import numpy as np

from . import prng
from .hmc import VELOCITY_VERLET, Metric, integrator_step, safe_energy_diff

F = np.float32
_NINF = F(-np.inf)


def _eps_col(step_size, C):
    eps = np.asarray(step_size, F)
    return (eps[:, None] if eps.ndim == 1 else np.full((C, 1), eps, F)).astype(F)


def _where(mask, a, b):
    return np.where(mask[:, None] if np.ndim(a) == 2 else mask, a, b).astype(F)


def num_steps_to_uturn(target, metric, q, p, g, eps, max_num_steps, coefficients=VELOCITY_VERLET, margin=None):
    """U(theta, rho) of every chain: steps until dot(theta_n - theta_0, rho_n) < 0 (raw momentum) or max_num_steps.
    margin (optional [C], updated in place): the smallest |dot| / (||theta_n - theta_0|| ||rho_n||) the rollout saw, a
    value near 0 marking a float tie."""
    C = q.shape[0]
    q0 = q
    n = np.zeros(C, np.int64)
    done = np.zeros(C, bool)
    with np.errstate(all="ignore"):
        while True:
            active = ~done & (n < max_num_steps)
            if not active.any():
                return n
            q1, p1, _, g1 = integrator_step(target, metric, q, p, g, eps, coefficients)
            q, p, g = _where(active, q1, q), _where(active, p1, p), _where(active, g1, g)
            n += active
            delta = (q - q0).astype(F)
            dot = np.sum(delta * p, axis=-1, dtype=F)
            if margin is not None:
                rel = np.abs(np.sum(delta.astype(np.float64) * p, -1)) / np.maximum(
                    np.linalg.norm(delta.astype(np.float64), axis=-1) * np.linalg.norm(p.astype(np.float64), axis=-1),
                    1e-300)
                margin[active] = np.minimum(margin[active], rel[active])
            done |= active & (dot < 0)


def step_distribution(u, path_fraction):
    """(lo, width) of trajectory_length.py:295-301: lo = max(1, floor(psi * U)) in float32."""
    lo = np.maximum(1, np.floor(F(path_fraction) * np.asarray(u).astype(F)).astype(np.int64))
    return lo, np.asarray(u) - lo + 1


def integrate_per_chain(target, metric, q, p, logp, g, eps, steps, coefficients=VELOCITY_VERLET):
    """steps[c] integrator steps for chain c (static_integration, chain by chain in lock step)."""
    with np.errstate(all="ignore"):
        for i in range(int(np.max(steps, initial=0))):
            act = steps > i
            q1, p1, lp1, g1 = integrator_step(target, metric, q, p, g, eps, coefficients)
            q, p, g, logp = _where(act, q1, q), _where(act, p1, p), _where(act, g1, g), _where(act, lp1, logp)
    return q, p, logp, g


def select_step_index(target, metric, q, p, logp, g, eps0, log_a, log_b, num_integration_steps, max_search_steps,
                      asymmetric=False, coefficients=VELOCITY_VERLET, margin=None):
    """The selector mu (step_size.py:184-289) of every chain from (q, p, logp, g): (step_index, search_exhausted).
    margin (optional [C], updated in place): the smallest distance of a compared |ell| (ell) to |log a| or |log b|."""
    C = q.shape[0]
    e_start = (-logp + metric.kinetic_energy(p)).astype(F)
    j = np.zeros(C, np.int64)
    v = np.zeros(C, np.int64)
    term = np.zeros(C, bool)
    la, lb = np.abs(log_a), np.abs(log_b)
    with np.errstate(all="ignore"):
        for it in range(max_search_steps + 1):
            active = ~term
            if not active.any():
                break
            tj = j if it == 0 else j + v
            eps = (eps0 * np.ldexp(F(1.0), tj.astype(np.int32))[:, None]).astype(F)
            q1, p1, lp1, _ = integrate_per_chain(target, metric, q, p, logp, g, eps, np.full(C, num_integration_steps),
                                                 coefficients)
            p1 = (F(-1.0) * p1).astype(F)
            ell = safe_energy_diff(e_start, (-lp1 + metric.kinetic_energy(p1)).astype(F))
            if not asymmetric:
                expand, shrink = np.abs(ell) < lb, np.abs(ell) > la
            else:
                expand, shrink = ell >= log_b, ell <= log_a
            vn = np.where(expand, 1, np.where(shrink, -1, 0)) if it == 0 else v
            if not asymmetric:
                te, ts = (vn == 1) & (np.abs(ell) >= lb), (vn == -1) & (np.abs(ell) <= la)
            else:
                te, ts = (vn == 1) & (ell < log_b), (vn == -1) & (ell > log_a)
            tn = (vn == 0) if it == 0 else (te | ts)
            if margin is not None:
                x = np.abs(ell) if not asymmetric else ell
                m = np.minimum(np.abs(x - (la if not asymmetric else log_a)), np.abs(x - (lb if not asymmetric else log_b)))
                margin[active] = np.minimum(margin[active], np.nan_to_num(m, nan=np.inf)[active])
            j = np.where(active, tj, j)
            v = np.where(active, vn, v)
            term = np.where(active, tn, term)
    exhausted = ~term & (v != 0)
    return np.where(term & (v == 1), j - 1, j), exhausted


def gist_kernel(keys, state, target, step_size, inverse_mass_matrix, instance="trajectory_length", path_fraction=0.5,
                max_num_steps=1024, num_integration_steps=1, criterion="symmetric", max_search_steps=10,
                divergence_threshold=1000.0, coefficients=VELOCITY_VERLET, margins=None):
    """One GIST transition for every chain.  keys uint32 [C, 2] (per-chain rng_key).  Returns (new_state, info) with info a
    dict of the bjx_gist_info fields (forward / reverse: U and N, or j and j_rev; rejected: is_no_return_rejected or
    search_exhausted).  margins (optional [C]): the tie margins of the instance's decisions (see the two helpers)."""
    metric = inverse_mass_matrix if isinstance(inverse_mass_matrix, Metric) else Metric(inverse_mass_matrix)
    q0, logp0, g0 = (np.asarray(x, F) for x in state)
    C, D = q0.shape
    ks = prng.split(keys, 3)                                           # _seam.py:163
    key_momentum, key_tuning, key_accept = ks[:, 0], ks[:, 1], ks[:, 2]
    p0 = metric.sample_momentum(key_momentum, D)                       # _seam.py:166
    eps0 = _eps_col(step_size, C)
    info = {}
    with np.errstate(all="ignore"):
        if instance == "trajectory_length":
            fwd = num_steps_to_uturn(target, metric, q0, p0, g0, eps0, max_num_steps, coefficients, margins)
            lo, w_fwd = step_distribution(fwd, path_fraction)
            L = np.array([int(prng.randint(key_tuning[c], (), int(lo[c]), int(fwd[c]) + 1)) for c in range(C)])
            q1, p1, logp1, g1 = integrate_per_chain(target, metric, q0, p0, logp0, g0, eps0, L, coefficients)
            p1 = (F(-1.0) * p1).astype(F)
            rev = num_steps_to_uturn(target, metric, q1, p1, g1, eps0, max_num_steps, coefficients, margins)
            lo_r, w_rev = step_distribution(rev, path_fraction)
            inside = (L >= lo_r) & (L <= rev)
            log_ratio = np.where(inside, (np.log(w_fwd.astype(F)) - np.log(w_rev.astype(F))).astype(F), _NINF).astype(F)
            info.update(num_integration_steps=L, forward=fwd, reverse=rev, rejected=~inside)
        elif instance == "step_size":
            if criterion not in ("symmetric", "asymmetric"):
                raise ValueError(f"criterion must be 'symmetric' or 'asymmetric', got {criterion!r}")
            asym = criterion == "asymmetric"
            u = prng.uniform(key_tuning, (2,))                             # step_size.py:296-298
            a, b = np.minimum(u[:, 0], u[:, 1]), np.maximum(u[:, 0], u[:, 1])
            log_a, log_b = np.log(a).astype(F), np.log(b).astype(F)
            j, ex_f = select_step_index(target, metric, q0, p0, logp0, g0, eps0, log_a, log_b, num_integration_steps,
                                        max_search_steps, asym, coefficients, margins)
            eps = (eps0 * np.ldexp(F(1.0), j.astype(np.int32))[:, None]).astype(F)
            q1, p1, logp1, g1 = integrate_per_chain(target, metric, q0, p0, logp0, g0, eps,
                                                    np.full(C, num_integration_steps), coefficients)
            p1 = (F(-1.0) * p1).astype(F)
            j_rev, ex_r = select_step_index(target, metric, q1, p1, logp1, g1, eps0, log_a, log_b, num_integration_steps,
                                            max_search_steps, asym, coefficients, margins)
            exhausted = ex_f | ex_r
            log_ratio = np.where((j_rev == j) & ~exhausted, F(0.0), _NINF).astype(F)
            info.update(num_integration_steps=np.full(C, num_integration_steps), forward=j, reverse=j_rev,
                        rejected=exhausted, a=a, b=b, step_size=eps[:, 0])
        else:
            raise ValueError(instance)
        e0 = (-logp0 + metric.kinetic_energy(p0)).astype(F)            # _seam.py:179
        e1 = (-logp1 + metric.kinetic_energy(p1)).astype(F)
        delta = safe_energy_diff(e0, e1)
        is_div = (-delta) > F(divergence_threshold)
        acc_prob = np.exp(np.minimum((delta + log_ratio).astype(F), F(0.0))).astype(F)   # _seam.py:186-187
    acc = prng.uniform(key_accept) < acc_prob
    new = (_where(acc, q1, q0), _where(acc, logp1, logp0), _where(acc, g1, g0))
    info.update(momentum=p0, acceptance_rate=acc_prob, is_accepted=acc, is_divergent=is_div, energy=e1,
                proposal=(q1, p1, logp1, g1))
    return new, info
