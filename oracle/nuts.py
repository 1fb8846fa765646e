"""Restatement of BlackJAX's iterative NUTS (batched over chains with masks) and of the
recursive tree builder that the reference keeps as its own second oracle.

TEST INFRASTRUCTURE (see oracle/__init__.py).  float32; per-chain results equal the
un-batched reference program (what ``jax.vmap(kernel)`` computes).

Follows:
* kernel / propose        blackjax/mcmc/nuts.py:113-145, :278-319
* tree doubling           blackjax/mcmc/trajectory.py:616-725 (dynamic_multiplicative_expansion)
* sub-tree                blackjax/mcmc/trajectory.py:273-393 (dynamic_progressive_integration)
* recursive builder       blackjax/mcmc/trajectory.py:398-560 (dynamic_recursive_integration)
* proposals               blackjax/mcmc/proposal.py:51-103 (generator), :118-143 (uniform), :146-176 (biased)
* termination             blackjax/mcmc/termination.py:31-106 (iterative_uturn_numpyro)
"""
from typing import NamedTuple

import numpy as np

from . import prng
from .hmc import F, HMCState, Metric, integrator_step, safe_energy_diff, VELOCITY_VERLET


def logaddexp(a, b):
    """jnp.logaddexp float32 semantics (NaN delta -> a + b)."""
    a = np.asarray(a, F)
    b = np.asarray(b, F)
    with np.errstate(invalid="ignore", over="ignore"):
        amax = np.maximum(a, b)
        delta = a - b
        r = amax + np.log1p(np.exp(-np.abs(delta))).astype(F)
        return np.where(np.isnan(delta), a + b, r).astype(F)


def expit(x):
    with np.errstate(over="ignore", invalid="ignore"):
        return (F(1.0) / (F(1.0) + np.exp(-np.asarray(x, F)))).astype(F)


def leaf_idx_to_ckpt_idxs(n):
    """termination.py:75-84."""
    n = int(n)
    idx_max = bin(n >> 1).count("1")
    num_subtrees = bin(((~n) & (n + 1)) - 1).count("1")
    return idx_max - num_subtrees + 1, idx_max


def is_iterative_turning(metric, ckpt_p, ckpt_sum, idx_min, idx_max, p_sum, p, margin=None):
    """termination.py:86-104 for ONE chain (ckpt arrays [depth, D]; ``metric`` is that chain's, see
    ``Metric.chain``).  ``margin``: 1-element array, lowered to the
    smallest relative distance of any evaluated U-turn product from its decision boundary (test aid)."""
    i = idx_max
    turning = False
    while i >= idx_min and not turning:
        sub = (p_sum - ckpt_sum[i] + ckpt_p[i]).astype(F)
        turning = bool(metric.is_turning(ckpt_p[i][None], p[None], sub[None])[0])
        if margin is not None:
            margin[0] = min(margin[0], float(metric.turning_margin(ckpt_p[i][None], p[None], sub[None])[0]))
        i -= 1
    return turning


class NUTSInfo(NamedTuple):
    momentum: np.ndarray
    is_divergent: np.ndarray
    is_turning: np.ndarray
    energy: np.ndarray
    trajectory_leftmost_state: tuple
    trajectory_rightmost_state: tuple
    num_trajectory_expansions: np.ndarray
    num_integration_steps: np.ndarray
    acceptance_rate: np.ndarray


def _sel(mask, a, b):
    m = mask if np.ndim(a) == 1 else mask[:, None]
    return np.where(m, a, b).astype(np.asarray(a).dtype)


def _lower(margins, mask, values):
    """margins[mask] = min(margins[mask], values[mask]) (NaNs ignored)."""
    if margins is None:
        return
    v = np.where(mask & np.isfinite(values), values, np.inf)
    np.minimum(margins, v, out=margins)


def subtree(target, metric, keys, q, p, logp, g, direction, ckpt_p, ckpt_sum, max_num_steps,
            eps, h0, run, divergence_threshold=1000.0, coefficients=VELOCITY_VERLET, margins=None):
    """dynamic_progressive_integration for all chains flagged ``run`` (bool[C]).

    Returns dict with the sub-tree's last leaf (q,p,logp,g), first leaf, momentum_sum,
    num_states, proposal (q,g,logp,energy,weight,slpa), is_diverging, has_terminated.
    ckpt_p / ckpt_sum ([C, depth, D]) are updated in place (threaded termination state).
    """
    C, D = q.shape
    eps_dir = (direction.astype(F) * np.asarray(eps, F))[:, None] if np.ndim(eps) == 0 \
        else (direction.astype(F) * np.asarray(eps, F))[:, None]
    cur = [q.copy(), p.copy(), logp.copy(), g.copy()]
    first = [q.copy(), p.copy(), logp.copy(), g.copy()]
    p_sum = p.copy()                                   # placeholder trajectory (:357-360)
    n = np.zeros(C, np.int32)
    # placeholder proposal = generate_proposal(H0, initial_state) (:356)
    e_init = (-logp + metric.kinetic_energy(p)).astype(F)
    w_init = safe_energy_diff(h0, e_init)
    prop = dict(q=q.copy(), g=g.copy(), logp=logp.copy(), energy=e_init, weight=w_init,
                slpa=np.minimum(w_init, F(0.0)).astype(F))
    is_div = np.zeros(C, bool)
    has_term = np.zeros(C, bool)
    act = run.copy()
    for i in range(int(max_num_steps)):
        if not act.any():
            break
        pk = prng.fold_in(keys, i)                                           # :321
        nq, np_, nlogp, ng = integrator_step(target, metric, cur[0], cur[1], cur[3], eps_dir,
                                             coefficients)                    # :323
        e_new = (-nlogp + metric.kinetic_energy(np_)).astype(F)
        w_new = safe_energy_diff(h0, e_new)                                  # proposal.py:94-98
        slpa_new = np.minimum(w_new, F(0.0)).astype(F)
        div_new = (-w_new) > F(divergence_threshold)                         # :325
        with np.errstate(invalid="ignore"):
            _lower(margins, act, np.abs(-w_new.astype(np.float64) - divergence_threshold) / divergence_threshold)
        if i == 0:                                                           # :329-334
            new_sum = np_.copy()
            acc = np.ones(C, bool)
            w_tot, slpa_tot = w_new, slpa_new
        else:                                                                # :335-338
            new_sum = (p_sum + np_).astype(F)
            with np.errstate(invalid="ignore"):
                p_accept = expit(w_new - prop["weight"])
            u_leaf = prng.uniform(pk)
            acc = u_leaf < p_accept
            _lower(margins, act, np.abs(u_leaf.astype(np.float64) - p_accept))
            w_tot = logaddexp(prop["weight"], w_new)
            slpa_tot = logaddexp(prop["slpa"], slpa_new)
        idx_min, idx_max = leaf_idx_to_ckpt_idxs(i)
        turning = np.zeros(C, bool)
        for c in np.nonzero(act)[0]:
            if i % 2 == 0:                                                   # termination.py:66-72
                ckpt_p[c, idx_max] = np_[c]
                ckpt_sum[c, idx_max] = new_sum[c]
            m1 = None if margins is None else margins[c:c + 1]
            # chain c's own metric: a per-chain metric batched against one chain's vectors would broadcast the
            # chain's momenta over every chain's inverse mass
            turning[c] = is_iterative_turning(metric.chain(c), ckpt_p[c], ckpt_sum[c], idx_min, idx_max,
                                              new_sum[c], np_[c], m1)
        # commit for active chains only
        for k, v in zip(range(4), (nq, np_, nlogp, ng)):
            cur[k] = _sel(act, v, cur[k])
        if i == 0:
            for k, v in zip(range(4), (nq, np_, nlogp, ng)):
                first[k] = _sel(act, v, first[k])
        p_sum = _sel(act, new_sum, p_sum)
        n = np.where(act, n + 1, n).astype(np.int32)
        take = act & acc
        prop["q"] = _sel(take, nq, prop["q"])
        prop["g"] = _sel(take, ng, prop["g"])
        prop["logp"] = _sel(take, nlogp, prop["logp"])
        prop["energy"] = _sel(take, e_new, prop["energy"])
        prop["weight"] = _sel(act, w_tot, prop["weight"])
        prop["slpa"] = _sel(act, slpa_tot, prop["slpa"])
        is_div = np.where(act, div_new, is_div)
        has_term = np.where(act, turning, has_term)
        act = act & ~div_new & ~turning
    return dict(last=cur, first=first, p_sum=p_sum, n=n, prop=prop, is_div=is_div, has_term=has_term)


def nuts_kernel(keys, state, target, step_size, inverse_mass_matrix, max_num_doublings=10,
                divergence_threshold=1000.0, coefficients=VELOCITY_VERLET, momentum=None,
                key_integrator=None, margins=None):
    """One NUTS transition for every chain.  keys uint32[C,2].  ``margins`` (test aid): float64[C] initialised to inf,
    lowered in place to each chain's smallest decision margin -- |u - p| of every multinomial / biased draw, the
    relative distance of every U-turn product from 0 and of -delta from the divergence threshold; a chain whose
    device result differs from this oracle by float rounding must show a margin near 0 (a tie)."""
    metric = inverse_mass_matrix if isinstance(inverse_mass_matrix, Metric) else Metric(inverse_mass_matrix)
    q0, logp0, g0 = (np.asarray(a, F) for a in state)
    C, D = q0.shape
    if key_integrator is None:
        ks = prng.split(keys, 2)                                             # nuts.py:133
        key_momentum, key_integrator = ks[:, 0], ks[:, 1]
        p0 = metric.sample_momentum(key_momentum, D)                          # nuts.py:136
    else:
        p0 = np.asarray(momentum, F)
    eps = np.asarray(step_size, F)
    h0 = (-logp0 + metric.kinetic_energy(p0)).astype(F)                      # nuts.py:282
    ckpt_p = np.zeros((C, max_num_doublings, D), F)                          # termination.py:46-54
    ckpt_sum = np.zeros((C, max_num_doublings, D), F)
    left = [q0.copy(), p0.copy(), logp0.copy(), g0.copy()]
    right = [q0.copy(), p0.copy(), logp0.copy(), g0.copy()]
    p_sum = p0.copy()                                                        # nuts.py:288-293
    n_states = np.zeros(C, np.int32)
    prop = dict(q=q0.copy(), g=g0.copy(), logp=logp0.copy(), energy=h0.copy(),
                weight=np.zeros(C, F), slpa=np.full(C, -np.inf, F))          # nuts.py:283-285
    step = np.zeros(C, np.int32)
    is_div = np.zeros(C, bool)
    is_turn = np.zeros(C, bool)
    for d in range(int(max_num_doublings)):
        run = (step < max_num_doublings) & ~is_div & ~is_turn                # trajectory.py:622-630
        if not run.any():
            break
        subkey = prng.fold_in(key_integrator, d)                             # :645 (step == d for running chains)
        k3 = prng.split(subkey, 3)                                           # :646
        direction_key, trajectory_key, proposal_key = k3[:, 0], k3[:, 1], k3[:, 2]
        direction = np.where(prng.bernoulli(direction_key), 1, -1).astype(np.int32)  # :650
        fwd = direction > 0
        start = [_sel(fwd, r, l) for r, l in zip(right, left)]               # :651-655
        sub = subtree(target, metric, trajectory_key, start[0], start[1], start[2], start[3],
                      direction, ckpt_p, ckpt_sum, 2 ** d, eps, h0, run,
                      divergence_threshold, coefficients, margins)           # :662-670
        sprop = sub["prop"]
        bad = sub["is_div"] | sub["has_term"]
        # :678-694 proposal update
        with np.errstate(invalid="ignore", over="ignore"):
            p_accept = np.minimum(np.exp((sprop["weight"] - prop["weight"]).astype(F)).astype(F), F(1.0))
        u_prop = prng.uniform(proposal_key)
        acc = u_prop < p_accept                                              # proposal.py:155-156
        _lower(margins, run & ~bad, np.abs(u_prop.astype(np.float64) - p_accept))
        new_w = logaddexp(prop["weight"], sprop["weight"])
        new_slpa = logaddexp(prop["slpa"], sprop["slpa"])
        take = run & ~bad & acc
        for k in ("q", "g", "logp", "energy"):
            prop[k] = _sel(take, sprop[k], prop[k])
        prop["weight"] = _sel(run & ~bad, new_w, prop["weight"])
        prop["slpa"] = _sel(run, new_slpa, prop["slpa"])
        # :697-704 merge (the sub-tree's last leaf becomes the new endpoint)
        for k in range(4):
            right[k] = _sel(run & fwd, sub["last"][k], right[k])
            left[k] = _sel(run & ~fwd, sub["last"][k], left[k])
        p_sum = _sel(run, (p_sum + sub["p_sum"]).astype(F), p_sum)
        n_states = np.where(run, n_states + sub["n"], n_states).astype(np.int32)
        turning = metric.is_turning(left[1], right[1], p_sum)                # :706-710
        if margins is not None:
            _lower(margins, run, metric.turning_margin(left[1], right[1], p_sum))
        step = np.where(run, step + 1, step).astype(np.int32)
        is_div = np.where(run, sub["is_div"], is_div)
        is_turn = np.where(run, sub["has_term"] | turning, is_turn)          # :715
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        acc_rate = (np.exp(prop["slpa"]).astype(F) / n_states.astype(F)).astype(F)   # nuts.py:303-305
    new_state = HMCState(prop["q"], prop["logp"], prop["g"])
    info = NUTSInfo(p0, is_div, is_turn, prop["energy"], tuple(left), tuple(right), step, n_states, acc_rate)
    return new_state, info


# ----------------------------------------------------------------------------------------------
# Recursive builder (single chain), trajectory.py:398-560 -- used only to cross-check `subtree`.
# ----------------------------------------------------------------------------------------------
def recursive_subtree(target, metric, key, state, direction, tree_depth, eps, h0,
                      divergence_threshold=1000.0):
    """Returns (key, proposal dict, trajectory dict(left,right,p_sum,n), is_diverging, is_turning)."""
    q, p, logp, g = state
    if tree_depth == 0:
        nq, np_, nlogp, ng = integrator_step(target, metric, q[None], p[None], g[None],
                                             F(direction) * F(eps))
        nq, np_, nlogp, ng = nq[0], np_[0], nlogp[0], ng[0]
        e = F(-nlogp + metric.kinetic_energy(np_[None])[0])
        w = safe_energy_diff(np.asarray(h0, F), np.asarray(e, F))
        propo = dict(state=(nq, np_, nlogp, ng), energy=e, weight=F(w), slpa=F(min(w, 0.0)))
        tr = dict(left=(nq, np_, nlogp, ng), right=(nq, np_, nlogp, ng), p_sum=np_.copy(), n=1)
        return key, propo, tr, bool(-w > divergence_threshold), False
    key, propo, tr, is_div, is_turn = recursive_subtree(target, metric, key, state, direction,
                                                        tree_depth - 1, eps, h0, divergence_threshold)
    if (not is_div) and (not is_turn):
        start = tr["right"] if direction > 0 else tr["left"]
        key, npropo, ntr, is_div, is_turn = recursive_subtree(target, metric, key, start, direction,
                                                              tree_depth - 1, eps, h0, divergence_threshold)
        lt, rt = (tr, ntr) if direction > 0 else (ntr, tr)
        tr = dict(left=lt["left"], right=rt["right"], p_sum=(lt["p_sum"] + rt["p_sum"]).astype(F),
                  n=lt["n"] + rt["n"])
        if not is_turn:
            is_turn = bool(metric.is_turning(tr["left"][1][None], tr["right"][1][None], tr["p_sum"][None])[0])
        ks = prng.split(key, 2)
        key, proposal_key = ks[0], ks[1]
        with np.errstate(invalid="ignore"):
            p_accept = expit(F(npropo["weight"]) - F(propo["weight"]))
        acc = bool(prng.uniform(proposal_key) < p_accept)
        w = logaddexp(propo["weight"], npropo["weight"])
        s = logaddexp(propo["slpa"], npropo["slpa"])
        src = npropo if acc else propo
        propo = dict(state=src["state"], energy=src["energy"], weight=F(w), slpa=F(s))
    return key, propo, tr, is_div, is_turn
