"""MCLMC's L / step-size tuner, ``mclmc_find_L_and_step_size`` (blackjax/adaptation/mclmc_adaptation.py:42-399), with an
explicit chain axis.

Chains never interact in this tuner: what ``jax.vmap(mclmc_find_L_and_step_size)`` gives the reference, one
``(L, step_size, inverse_mass_matrix)`` per chain, is what this returns, each chain running the reference's single-chain
algorithm with its own key (``split(rng_key, n_global)[chain_offset + c]``, or the caller's ``[C, 2]`` keys).  All three
stages run on the device (libbjx ``bjx_mclmc_find_l_and_step_size``): the fused tuning step ``k_mclmc_tune``, plain MCLMC
transitions, and the per-chain ESS ``k_ess_chain``.  The returned parameters plug into ``blackjax.mclmc`` and
``sample_mclmc_native`` as they are: ``L`` and ``step_size`` are ``[C]``, ``inverse_mass_matrix`` is ``[C, D]``.
"""
from typing import NamedTuple

import torch

from .._engine import as_keys, get_engine
from .._lib import check, lib, ptr
from ..mcmc.hmc import IntegratorState

__all__ = ["MCLMCAdaptationState", "mclmc_find_L_and_step_size", "stage_lengths"]


class MCLMCAdaptationState(NamedTuple):
    """mclmc_adaptation.py:26-39, per chain: L [C], step_size [C], inverse_mass_matrix [C, D]."""

    L: torch.Tensor
    step_size: torch.Tensor
    inverse_mass_matrix: torch.Tensor


def stage_lengths(num_steps, frac_tune1, frac_tune2, frac_tune3, diagonal_preconditioning):
    """(n1, n2, readjust steps run, n3, returned step count) as the reference forms them (:180-203, :318-320, :356):
    Python's round (halves to even); the readjustment runs round(n2 / 3) steps when n2 > 1 and diagonal preconditioning
    is on, but the count adds n2 // 3 whenever it is on; stage 3 runs and counts only when n3 >= 2."""
    n1, n2, n3 = round(num_steps * frac_tune1), round(num_steps * frac_tune2), round(num_steps * frac_tune3)
    readjust = round(n2 / 3) if (n2 > 1 and diagonal_preconditioning) else 0
    count = n1 + n2 + (n2 // 3 if diagonal_preconditioning else 0) + (n3 if n3 >= 2 else 0)
    return n1, n2, readjust, n3, count


def _per_chain(x, shape, device):
    """A scalar, or an array that broadcasts to ``shape``, as a fresh float32 tensor of that shape."""
    t = torch.as_tensor(x, dtype=torch.float32, device=device)
    return t.broadcast_to(shape).contiguous().clone()


def mclmc_find_L_and_step_size(mclmc_kernel, num_steps, state, rng_key, logdensity_fn=None, frac_tune1=0.1,
                               frac_tune2=0.1, frac_tune3=0.1, desired_energy_var=5e-4, trust_in_estimate=1.5,
                               num_effective_samples=150, diagonal_preconditioning=True, params=None, l_factor=0.4, *,
                               max_history_bytes=1 << 31, divergences=None):
    """blackjax/adaptation/mclmc_adaptation.py:42-205 for every chain.

    ``mclmc_kernel`` must come from ``blackjax_b200.mclmc.build_kernel``: its integrator, energy cutoff and
    ``chain_offset`` are what the tuner runs with.  ``state`` is an MCLMC ``IntegratorState`` with positions
    ``[C, D]``; it is not modified.  ``params`` (optional) gives the initial parameters; scalars and ``[D]`` metrics
    broadcast to every chain.  Without it ``L = sqrt(D)``, ``step_size = sqrt(D) / 4`` and ``M^-1 = 1``.

    ``max_history_bytes`` bounds the position history of stage 3, which runs on slices of chains that fit it (the result
    does not depend on the slice size).  ``divergences`` (optional) is a ``uint8`` tensor ``[steps, C]`` that receives 1
    for every failed tuning step of stages 1 and 2 and of the readjustment, in that order (the reference's scan output);
    ``steps = n1 + n2 + readjust`` from :func:`stage_lengths`.

    Returns ``(IntegratorState, MCLMCAdaptationState, total number of tuning steps)``.
    """
    if logdensity_fn is None:
        raise ValueError("logdensity_fn is required. Pass the log-density function of the target distribution.")
    coefficients = getattr(mclmc_kernel, "coefficients", None)
    if coefficients is None or not hasattr(mclmc_kernel, "desired_energy_var_max_ratio"):
        raise TypeError("mclmc_kernel must be a kernel built by blackjax_b200.mclmc.build_kernel")
    from ..mcmc.mclmc import energy_cutoff
    q, p, logp, g = (t.clone() for t in state)
    C, D = q.shape
    dev = q.device
    eng = get_engine(q, logdensity_fn)
    if params is None:
        L0 = torch.sqrt(torch.tensor(float(D), dtype=torch.float32))
        params = MCLMCAdaptationState(L0, L0 * 0.25, 1.0)
    L = _per_chain(params.L, (C,), dev)
    step_size = _per_chain(params.step_size, (C,), dev)
    imm = _per_chain(params.inverse_mass_matrix, (C, D), dev)
    n1, n2, readjust, n3, count = stage_lengths(num_steps, frac_tune1, frac_tune2, frac_tune3, diagonal_preconditioning)
    if divergences is not None and (divergences.dtype != torch.uint8 or tuple(divergences.shape) != (n1 + n2 + readjust, C)
                                    or not divergences.is_contiguous()):
        raise ValueError(f"divergences must be a contiguous uint8 tensor of shape ({n1 + n2 + readjust}, {C})")
    eng.set_integrator(coefficients)
    # libbjx checks the configuration against the installed metric; the tuner itself runs with its own copy `imm`, which
    # it rewrites, so the engine's cached metric is dropped afterwards
    eng._tune_metric = imm.clone()
    eng.ensure_metric(eng._tune_metric, diagonal_only=True)
    keys = as_keys(rng_key, C, dev)
    eng._key_mode(keys, getattr(mclmc_kernel, "chain_offset", 0))
    try:
        check(lib().bjx_mclmc_find_l_and_step_size(
            eng.h, ptr(keys), ptr(q), ptr(p), ptr(logp), ptr(g), ptr(step_size), ptr(L), ptr(imm), n1, n2, readjust, n3,
            int(bool(diagonal_preconditioning)),
            energy_cutoff(D, mclmc_kernel.desired_energy_var_max_ratio, mclmc_kernel.desired_energy_var),
            float(desired_energy_var), float(trust_in_estimate), float(num_effective_samples), float(l_factor),
            int(max_history_bytes), ptr(divergences)), eng.h)
    finally:
        eng._imm_key = None
    return IntegratorState(q, p, logp, g), MCLMCAdaptationState(L, step_size, imm), count


def tune_step_(eng, keys, state, step_size, L, cutoff, adaptive, streaming, mask, desired_energy_var=5e-4,
               trust_in_estimate=1.5, num_effective_samples=150, chain_offset=0):
    """One tuning step (predictor + step, :223-301) in place, libbjx ``bjx_mclmc_tune_step``, on the engine's installed
    metric.  ``state`` = (q, p, logp, g); ``step_size`` [C]; ``adaptive`` = (time, x_average, step_size_max) [C] each;
    ``streaming`` = (total [C], moments [C, 2, D]) or None.  All are updated in place.  Returns success [C] (bool)."""
    q, p, logp, g = state
    keys = as_keys(keys, eng.C, eng.device)
    eng._key_mode(keys, chain_offset)
    L, L_dev = eng._eps(L, "L")
    total, moments = streaming if streaming is not None else (None, None)
    success = torch.empty(eng.C, dtype=torch.uint8, device=eng.device)
    check(lib().bjx_mclmc_tune_step(eng.h, ptr(keys), ptr(q), ptr(p), ptr(logp), ptr(g), ptr(step_size), L, ptr(L_dev),
                                    float(cutoff), *(ptr(t) for t in adaptive), ptr(total), ptr(moments), int(mask),
                                    float(desired_energy_var), float(trust_in_estimate), float(num_effective_samples),
                                    ptr(success)), eng.h)
    return success.bool()
