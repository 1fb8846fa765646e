"""Float32 restatement of MCLMC (blackjax/mcmc/mclmc.py, the isokinetic integrators of blackjax/mcmc/integrators.py:
372-600, generate_unit_vector of blackjax/util.py:94-113), batched over chains, on top of oracle/prng.py and the targets
of oracle/targets.py.  Every array is [C, D] (or [C] for per-chain scalars); each chain behaves like one jax.vmap lane.

Rounding follows the device kernel: the position update x + (eps c) * (sqrt(M^-1) u) is one fused multiply-add (as the
other oracles' FMA_CONTRACT), every other elementwise operation is one float32 rounding.
"""
import numpy as np

from . import prng as oprng

F = np.float32
TOL = F(1e-13)  # _normalized_flatten_array (integrators.py:374-376)


def _norm(x):
    return np.sqrt(np.sum(x * x, axis=-1, dtype=F)).astype(F)


def unit_vector(keys, D):
    """generate_unit_vector: normal(key, (D,)) / ||.||, one key [.., 2] per chain."""
    z = oprng.normal(keys, (D,))
    return (z / _norm(z)[..., None]).astype(F)


def partial_refresh(u, keys, step_size, L):
    """partially_refresh_momentum (integrators.py:543-572); step_size is eps / 2 at both call sites; L scalar or [C]."""
    D = u.shape[-1]
    L = np.broadcast_to(np.asarray(L, F), u.shape[:-1])
    step_size = np.broadcast_to(np.asarray(step_size, F), u.shape[:-1])
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        nu = np.sqrt(((np.exp((F(2.0) * step_size / L).astype(F)) - F(1.0)) / F(D)).astype(F)).astype(F)
        m = (u + nu[..., None] * oprng.normal(keys, (D,))).astype(F)
        new = (m / _norm(m)[..., None]).astype(F)
    return np.where(np.isinf(L)[..., None], u, new).astype(F)


def esh_update(u, g, sqrt_imm, a):
    """esh_dynamics_momentum_update_one_step (integrators.py:438-479) with step_size * coef = a [C] (or scalar).
    Returns (new unit momentum, kinetic-energy change of this stage)."""
    D = u.shape[-1]
    a = np.broadcast_to(np.asarray(a, F), u.shape[:-1])
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        gt = (g * sqrt_imm).astype(F)
        gn = _norm(gt)
        gh = np.where((gn > TOL)[..., None], gt / gn[..., None], gt).astype(F)
        proj = np.sum(u * gh, axis=-1, dtype=F)
        delta = ((a * gn).astype(F) / F(D - 1)).astype(F)
        zeta = np.exp(-delta).astype(F)
        omz = (F(1.0) - zeta).astype(F)
        b = ((F(1.0) + zeta) + proj * omz).astype(F)
        raw = ((gh * omz[..., None]) * b[..., None] + (F(2.0) * zeta)[..., None] * u).astype(F)
        rn = _norm(raw)
        new = np.where((rn > TOL)[..., None], raw / rn[..., None], raw).astype(F)
        dk = ((delta - F(np.log(2.0))) + np.log((F(1.0) + proj) + (F(1.0) - proj) * (zeta * zeta))).astype(F) * F(D - 1)
    return new, dk.astype(F)


def position_update(q, u, sqrt_imm, a):
    """euclidean_position_update_fn (integrators.py:191-205): x + (eps c) * forward_L(u), forward_L(u) = sqrt(M^-1) u."""
    a = np.broadcast_to(np.asarray(a, F), q.shape[:-1])
    kg = (u * sqrt_imm).astype(F)
    with np.errstate(over="ignore", invalid="ignore"):
        return (q.astype(np.float64) + a[..., None].astype(np.float64) * kg.astype(np.float64)).astype(F)


def isokinetic_step(q, u, logp, g, target, sqrt_imm, eps, coefficients):
    """One step of the isokinetic integrator with a palindromic table (generalized_two_stage_integrator,
    integrators.py:104-150).  Returns (q, u, logp, g, kinetic_change)."""
    eps = np.broadcast_to(np.asarray(eps, F), q.shape[:-1])
    dk_sum = np.zeros(q.shape[:-1], F)
    for i, c in enumerate(coefficients):
        a = (eps * F(c)).astype(F)
        if i % 2 == 0:
            u, dk = esh_update(u, g, sqrt_imm, a)
            dk_sum = (dk_sum + dk).astype(F)
        else:
            q = position_update(q, u, sqrt_imm, a)
            with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
                logp, g = target(q)
    return q, u, logp, g, dk_sum


class MCLMCInfo:
    def __init__(self, logdensity, kinetic_change, energy_change, nonans):
        self.logdensity, self.kinetic_change, self.energy_change, self.nonans = (
            logdensity, kinetic_change, energy_change, nonans)


def mclmc_kernel(keys, state, target, inverse_mass_matrix, L, step_size, coefficients, cutoff=np.inf):
    """mclmc.build_kernel(...).kernel (mclmc.py:104-143) for per-chain keys [C, 2].  state = (q, u, logp, g);
    inverse_mass_matrix [D] or [C, D]; L, step_size scalar or [C]; cutoff = sqrt(D * max_ratio * desired_energy_var)."""
    q0, u0, logp0, g0 = (np.asarray(x, F) for x in state)
    C, D = q0.shape
    sqrt_imm = np.sqrt(np.broadcast_to(np.asarray(inverse_mass_matrix, F), (C, D))).astype(F)
    eps = np.broadcast_to(np.asarray(step_size, F), (C,))
    k3 = oprng.split(keys, 3)
    kernel_key, cut_key, nan_key = k3[:, 0], k3[:, 1], k3[:, 2]
    k12 = oprng.split(kernel_key, 2)
    half = (eps * F(0.5)).astype(F)
    u = partial_refresh(u0, k12[:, 0], half, L)
    q, u, logp, g, kc = isokinetic_step(q0, u, logp0, g0, target, sqrt_imm, eps, coefficients)
    u = partial_refresh(u, k12[:, 1], half, L)
    with np.errstate(invalid="ignore", over="ignore"):
        ec = ((kc - logp).astype(F) + logp0).astype(F)
        high = np.abs(ec) > F(cutoff)
    q = np.where(high[:, None], q0, q)
    g = np.where(high[:, None], g0, g)
    logp = np.where(high, logp0, logp).astype(F)
    u = np.where(high[:, None], unit_vector(cut_key, D), u)
    kc = np.where(high, F(0), kc).astype(F)
    ec = np.where(high, F(0), ec).astype(F)
    nonans = np.all(np.isfinite(q), axis=1) & np.all(np.isfinite(u), axis=1) & np.isfinite(logp)
    bad = ~nonans
    q = np.where(bad[:, None], q0, q)
    g = np.where(bad[:, None], g0, g)
    logp = np.where(bad, logp0, logp).astype(F)
    u = np.where(bad[:, None], unit_vector(nan_key, D), u)
    kc = np.where(bad, F(0), kc).astype(F)
    ec = np.where(bad, F(0), ec).astype(F)
    return (q, u, logp, g), MCLMCInfo(logp, kc, ec, nonans)


def mclmc_init(position, target, keys):
    """mclmc.init (mclmc.py:55-66) for per-chain keys [C, 2]."""
    q = np.asarray(position, F)
    logp, g = target(q)
    return q, unit_vector(keys, q.shape[1]), logp, g

