"""Float32 restatement of adjusted MCLMC / MAMS (blackjax/mcmc/adjusted_mclmc.py, adjusted_mclmc_dynamic.py), batched over
chains, on top of oracle/mclmc.py (unit_vector, partial_refresh, isokinetic_step) and oracle/prng.py.  Every
chain has its own number of integration steps n (an array [C]); each chain behaves like one jax.vmap lane.

Key tree of one chain's key (adjusted_mclmc.py:86,232,255-263; integrators.py:577):
    key_momentum, key_integrator = split(key, 2)
    k_0 = key_integrator;  a_i, k_{i+1} = split(k_i) for step i = 0 .. n-1
    step i refreshes the momentum with split(a_i)[0] before and split(a_i)[1] after its integrator step
    the Metropolis uniform is uniform(k_n)  (= uniform(key_integrator) when n = 0)
"""
import numpy as np

from . import mclmc as om
from . import prng as oprng

F = np.float32


def rescale(mu):
    """adjusted_mclmc.py:281-288 in float32: s such that round(U * s + 0.5) has mean mu."""
    mu = F(mu)
    k = np.floor(F(2) * mu - F(1))
    x = k * (mu - F(0.5) * (k + F(1))) / (k + F(1) - mu)
    return F(k + x)


def steps_randint(keys):
    """The default step-count rule, jax.random.randint(key, (), 1, 10) (adjusted_mclmc_dynamic.py:55)."""
    return oprng.randint(keys, (), 1, 10).astype(np.int32)


def steps_uniform(keys, avg, min_steps=1):
    """max(ceil(uniform(key) * rescale(avg)), min_steps) (adjusted_mclmc_dynamic.py:234-238 with min_steps = 1; the
    reference's sampling tests use it unclipped, min_steps = 0)."""
    n = np.ceil((oprng.uniform(keys) * rescale(avg)).astype(F)).astype(np.int32)
    return np.maximum(n, min_steps).astype(np.int32)


def halton_sequence(i, max_bits=10):
    """The (i+1)-th element of the base-2 Halton sequence (dynamic_hmc.py:205-215), elementwise; exact in float32."""
    i = np.asarray(i, np.int64)
    b = 2 ** np.arange(max_bits, dtype=np.int64)
    return (np.mod((i[..., None] + 1) // b, 2).astype(F) * (F(0.5) / b.astype(F))).sum(-1, dtype=F)


def trajectory_length(t, mu):
    """adjusted_mclmc_dynamic.py:197-212."""
    return np.rint(F(0.5) + halton_sequence(t) * rescale(mu)).astype(np.int32)


class Info:
    """HMCInfo as adjusted_mclmc_proposal fills it (adjusted_mclmc.py:266-274), plus delta and the uniform drawn."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def adjusted_mclmc_kernel(keys, state, target, inverse_mass_matrix, step_size, num_integration_steps, coefficients,
                          L_proposal_factor=np.inf, divergence_threshold=1000.0):
    """adjusted_mclmc.build_kernel(...).kernel for per-chain keys [C, 2]; state = (q, logp, g); inverse_mass_matrix [D] or
    [C, D]; step_size scalar or [C]; num_integration_steps int or [C]."""
    q0, logp0, g0 = (np.asarray(x, F) for x in state)
    C, D = q0.shape
    sqrt_imm = np.sqrt(np.broadcast_to(np.asarray(inverse_mass_matrix, F), (C, D))).astype(F)
    eps = np.broadcast_to(np.asarray(step_size, F), (C,)).astype(F)
    n = np.broadcast_to(np.asarray(num_integration_steps, np.int32), (C,))
    with np.errstate(invalid="ignore", over="ignore"):
        L = (F(L_proposal_factor) * (n.astype(F) * eps).astype(F)).astype(F)
    km = oprng.split(keys, 2)
    u0 = om.unit_vector(km[:, 0], D)
    k = km[:, 1]
    half = (eps * F(0.5)).astype(F)
    q, u, logp, g = q0, u0, logp0, g0
    kinetic = (logp0 * F(0.0)).astype(F)
    for i in range(int(n.max(initial=0))):
        act = i < n
        ak = oprng.split(k, 2)
        a, k = ak[:, 0], np.where(act[:, None], ak[:, 1], k)
        r = oprng.split(a, 2)
        with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
            u1 = om.partial_refresh(u, r[:, 0], half, np.where(act, L, np.inf))
            q1, u1, logp1, g1, dk = om.isokinetic_step(q, u1, logp, g, target, sqrt_imm, eps, coefficients)
            u1 = om.partial_refresh(u1, r[:, 1], half, np.where(act, L, np.inf))
        q, u, g = (np.where(act[:, None], new, old) for new, old in ((q1, q), (u1, u), (g1, g)))
        logp = np.where(act, logp1, logp).astype(F)
        kinetic = np.where(act, (kinetic + dk).astype(F), kinetic).astype(F)
    with np.errstate(invalid="ignore", over="ignore"):
        delta = ((-logp0 + logp).astype(F) - kinetic).astype(F)
        delta = np.where(np.isnan(delta), F(-np.inf), delta).astype(F)
        is_div = -delta > F(divergence_threshold)
        p_acc = np.minimum(np.exp(delta), F(1)).astype(F)
    uni = oprng.uniform(k)
    acc = uni < p_acc
    new = (np.where(acc[:, None], q, q0), np.where(acc, logp, logp0).astype(F), np.where(acc[:, None], g, g0))
    info = Info(momentum=u0, acceptance_rate=p_acc, is_accepted=acc, is_divergent=is_div, energy=(-logp).astype(F),
                proposal=(q, u, logp, g), num_integration_steps=n.copy(), delta=delta, uniform=uni)
    return new, info


def dynamic_kernel(keys, state, target, inverse_mass_matrix, step_size, coefficients, steps_fn=steps_randint,
                   L_proposal_factor=np.inf, divergence_threshold=1000.0):
    """adjusted_mclmc_dynamic.build_kernel(...).kernel: state = (q, logp, g, random_generator_arg [C, 2]); steps_fn maps
    random_generator_arg to n [C]; the next random_generator_arg is split(key)[1]."""
    q, logp, g, rga = state
    n = steps_fn(rga)
    new, info = adjusted_mclmc_kernel(keys, (q, logp, g), target, inverse_mass_matrix, step_size, n, coefficients,
                                      L_proposal_factor, divergence_threshold)
    return (*new, oprng.split(rga, 2)[:, 1]), info
