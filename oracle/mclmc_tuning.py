"""Float32 restatement of MCLMC's L / step-size tuner (blackjax/adaptation/mclmc_adaptation.py:42-452, with
incremental_value_update of blackjax/util.py:287-319), batched over independent chains, on top of oracle/mclmc.mclmc_kernel,
oracle/prng.py and oracle/diagnostics.effective_sample_size.  Every chain behaves like one jax.vmap lane of the reference.

The step-size clip.  The reference writes it as (eps' < eps_max) * eps' + (eps' > eps_max) * eps_max and starts from
eps_max = inf.  Under literal IEEE arithmetic the first step would give 0 * inf = NaN, every later step size would be NaN,
and the reference's own tests (tests/mcmc/test_mclmc_nan_fix_969.py: final step sizes in (0.1, 10)) could not pass.  XLA's
algebraic simplifier rewrites a multiply by a converted predicate into a select, so what runs is: eps' where eps' < eps_max,
eps_max where eps' > eps_max, 0 where they are equal or eps' is NaN.  That reading rests on the rewrite and on those tests'
outcome; it has not been checked against a live JAX run.
"""
import numpy as np

from . import mclmc as mo
from . import prng as oprng
from .diagnostics import effective_sample_size

F = np.float32


def stage_lengths(num_steps, frac_tune1, frac_tune2, frac_tune3, diagonal_preconditioning):
    """(n1, n2, readjust steps run, n3, returned count): mclmc_adaptation.py:180-203, :318-320, :356."""
    n1, n2, n3 = round(num_steps * frac_tune1), round(num_steps * frac_tune2), round(num_steps * frac_tune3)
    readjust = round(n2 / 3) if (n2 > 1 and diagonal_preconditioning) else 0
    count = n1 + n2 + diagonal_preconditioning * (n2 // 3) + (n3 if n3 >= 2 else 0)
    return n1, n2, readjust, n3, count


def clip_step_size(new, eps_max):
    """The reference's clip as XLA evaluates it (see the module docstring)."""
    new, eps_max = np.asarray(new, F), np.asarray(eps_max, F)
    return np.where(new < eps_max, new, np.where(new > eps_max, eps_max, F(0))).astype(F)


def safediv(x, y):
    """util.py:287-288: 0 exactly where the numerator is 0."""
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(x == 0, F(0), (x / y).astype(F)).astype(F)


def incremental_value_update(x, total, moments, weight):
    """util.py:291-319 on expectation (x, x^2): moments [C, 2, D], total / weight [C].  (total av + w exp) / (total + w)
    is evaluated even when w = 0: it can move av by one ulp."""
    w = weight[:, None]
    exp = np.stack([x, (x * x).astype(F)], axis=1)
    num = ((total[:, None, None] * moments).astype(F) + (w[:, None] * exp).astype(F)).astype(F)
    den = (total + weight).astype(F)
    return (total + weight).astype(F), safediv(num, den[:, None, None])


class Constants:
    """The predictor's constants as the reference forms them: Python floats, float32 inside the jnp expressions."""

    def __init__(self, dim, desired_energy_var=5e-4, trust_in_estimate=1.5, num_effective_samples=150):
        self.dim_eev = F(dim * desired_energy_var)
        self.trust6 = F(6.0 * trust_in_estimate)
        self.decay = F((num_effective_samples - 1.0) / (num_effective_samples + 1.0))


def predictor(energy_change, success, eps, adaptive, k):
    """The step-size update of predictor (:243-272) after the transition: (new step size, (time, x_average,
    step_size_max)).  A failed step counts with energy change 0 and sets step_size_max = 0.8 eps."""
    time, x_avg, eps_max = (np.asarray(a, F) for a in adaptive)
    eps_max = np.where(success, eps_max, (eps * F(0.8)).astype(F)).astype(F)
    ec = np.where(success, energy_change, F(0)).astype(F)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        xi = ((ec * ec).astype(F) / k.dim_eev + F(1e-8)).astype(F)
        lx = (np.log(xi).astype(F) / k.trust6).astype(F)
        w = np.exp((F(-0.5) * (lx * lx).astype(F)).astype(F)).astype(F)
        x_avg = ((k.decay * x_avg).astype(F) + (w * (xi / np.power(eps, F(6.0)).astype(F)).astype(F)).astype(F)).astype(F)
        time = ((k.decay * time).astype(F) + w).astype(F)
        eps_new = np.power((x_avg / time).astype(F), F(-1.0 / 6.0)).astype(F)
    return clip_step_size(eps_new, eps_max), (time, x_avg, eps_max)


def tune_step(keys, state, target, imm, L, eps, adaptive, streaming, mask, coefficients, cutoff, k):
    """One scan step (predictor + step, :223-301) for per-chain step keys [C, 2].  adaptive = (time, x_average,
    step_size_max) [C]; streaming = (total [C], moments [C, 2, D]).  Returns (state, eps', adaptive, streaming, success)."""
    q0, u0, logp0, g0 = (np.asarray(x, F) for x in state)
    C, D = q0.shape
    eps = np.broadcast_to(np.asarray(eps, F), (C,)).astype(F)
    time, x_avg, eps_max = (np.asarray(a, F) for a in adaptive)
    kk = oprng.split(keys, 2)
    rng_key, nan_key = kk[:, 0], kk[:, 1]
    (q, u, logp, g), info = mo.mclmc_kernel(rng_key, (q0, u0, logp0, g0), target, imm, L, eps, coefficients, cutoff)
    with np.errstate(invalid="ignore"):
        success = info.nonans & np.isfinite(info.energy_change)
    s1, s2 = success[:, None], success
    q_n = np.where(s1, np.nan_to_num(q), q0).astype(F)
    u_n = np.where(s1, np.nan_to_num(u), u0).astype(F)
    logp_n = np.where(s2, np.nan_to_num(logp), logp0).astype(F)
    g_n = np.where(s1, np.nan_to_num(g), g0).astype(F)
    u_n = np.where(np.isnan(logp)[:, None], mo.unit_vector(nan_key, D), u_n).astype(F)
    eps_new, (time, x_avg, eps_max) = predictor(info.energy_change, success, eps, (time, x_avg, eps_max), k)
    total, moments = streaming
    weight = (F(mask) * success.astype(F) * eps_new).astype(F)
    total, moments = incremental_value_update(q_n, np.asarray(total, F), np.asarray(moments, F), weight)
    return (q_n, u_n, logp_n, g_n), eps_new, (time, x_avg, eps_max), (total, moments), success


def _run_steps(base_keys, n, mask_from, state, target, imm, L, eps, coefficients, cutoff, k):
    C, D = state[0].shape
    adaptive = (np.zeros(C, F), np.zeros(C, F), np.full(C, np.inf, F))
    streaming = (np.zeros(C, F), np.zeros((C, 2, D), F))
    div = []
    for t in range(n):
        step_keys = oprng.fold_in(base_keys, t)
        state, eps, adaptive, streaming, success = tune_step(step_keys, state, target, imm, L, eps, adaptive, streaming,
                                                             float(t >= mask_from), coefficients, cutoff, k)
        div.append(~success)
    return state, eps, streaming, div


def find_L_and_step_size(chain_keys, num_steps, state, target, coefficients, cutoff=np.inf, frac_tune1=0.1,
                         frac_tune2=0.1, frac_tune3=0.1, desired_energy_var=5e-4, trust_in_estimate=1.5,
                         num_effective_samples=150, diagonal_preconditioning=True, params=None, l_factor=0.4):
    """mclmc_find_L_and_step_size (:42-205) for every chain: chain_keys [C, 2] are the chains' own keys.  params =
    (L, step_size, inverse_mass_matrix) broadcastable to [C], [C], [C, D].  Returns (state, (L, eps, imm), count,
    divergence flags [steps, C])."""
    state = tuple(np.asarray(x, F) for x in state)
    C, D = state[0].shape
    if params is None:
        L0 = np.sqrt(F(D)).astype(F)
        params = (L0, (L0 * F(0.25)).astype(F), F(1))
    L = np.broadcast_to(np.asarray(params[0], F), (C,)).copy()
    eps = np.broadcast_to(np.asarray(params[1], F), (C,)).copy()
    imm = np.broadcast_to(np.asarray(params[2], F), (C, D)).copy()
    k = Constants(D, desired_energy_var, trust_in_estimate, num_effective_samples)
    n1, n2, readjust, n3, count = stage_lengths(num_steps, frac_tune1, frac_tune2, frac_tune3, diagonal_preconditioning)
    parts = oprng.split(chain_keys, 2)
    part1, part2 = parts[:, 0], parts[:, 1]
    state, eps, (_, moments), div = _run_steps(part1, n1 + n2, n1, state, target, imm, L, eps, coefficients, cutoff, k)
    L_out = L
    if n2 > 1:  # :340-360
        var = (moments[:, 1] - (moments[:, 0] * moments[:, 0]).astype(F)).astype(F)
        L_out = np.sqrt(np.sum(var, axis=1, dtype=F)).astype(F)
        if diagonal_preconditioning:
            imm = var
            L_out = np.full(C, np.sqrt(F(D)), F)
            final_key = oprng.fold_in(part1, n1 + n2)
            state, eps, _, div2 = _run_steps(final_key, readjust, 0, state, target, imm, L, eps, coefficients, cutoff, k)
            div += div2
    L = L_out
    if n3 >= 2:  # :367-399
        hist = []
        for t in range(n3):
            state, _ = mo.mclmc_kernel(oprng.fold_in(part2, t), state, target, imm, L, eps, coefficients, cutoff)
            hist.append(state[0])
        hist = np.stack(hist)  # [n3, C, D]
        ess = np.stack([np.atleast_1d(effective_sample_size(hist[:, c][None], chain_axis=0, sample_axis=1))
                        for c in range(C)]).astype(F)
        with np.errstate(divide="ignore"):
            ratio = (F(n3) / ess).astype(F)
        L = ((F(l_factor) * eps).astype(F) * np.mean(ratio, axis=1, dtype=F)).astype(F)
    return state, (L, eps, imm), count, (np.stack(div) if div else np.zeros((0, C), bool))
