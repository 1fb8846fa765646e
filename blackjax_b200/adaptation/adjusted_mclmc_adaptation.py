"""Adjusted MCLMC's tuner, ``adjusted_mclmc_find_L_and_step_size`` (blackjax/adaptation/adjusted_mclmc_adaptation.py:26-507),
with an explicit chain axis.

Chains never interact in this tuner: what ``jax.vmap(adjusted_mclmc_find_L_and_step_size)`` gives the reference, one
``(L, step_size, inverse_mass_matrix)`` per chain, is what this returns, each chain running the reference's single-chain
algorithm with its own key (``split(rng_key, n_global)[chain_offset + c]``, or the caller's ``[C, 2]`` keys).  Every
window, both dual-averaging passes, the variance step and stage 3 run on the device (libbjx
``bjx_adjusted_mclmc_find_l_and_step_size``): the fused tuning step ``k_amclmc_tune``, plain adjusted MCLMC transitions and
the per-chain ESS ``k_ess_chain``.  ``L / step_size`` of the result is a per-chain ``[C]`` tensor that
``adjusted_mclmc(num_integration_steps=...)``, ``adjusted_mclmc_dynamic(integration_steps_params=(...,))`` and
``sample_adjusted_mclmc_native`` take as it is.
"""
import torch

from .._engine import as_keys, get_engine
from .._lib import AMCLMC_STEPS_FIXED, check, lib, ptr
from ..mcmc.dynamic_hmc import DynamicHMCState
from ..mcmc.hmc import HMCState
from .mclmc_adaptation import MCLMCAdaptationState, _per_chain

__all__ = ["adjusted_mclmc_find_L_and_step_size", "stage_lengths"]

L_FACTOR = 0.5  # adjusted_mclmc_make_adaptation_L's l_factor as the top-level function passes it (:167)


def stage_lengths(num_steps, frac_tune1, frac_tune2, frac_tune3, num_windows=1):
    """(n1, n2, n3) as the reference forms them: frac /= num_windows (:114-116), then int() truncation (:328-330, :445);
    stage 3 runs only when frac_tune3 != 0."""
    f1, f2, f3 = frac_tune1 / num_windows, frac_tune2 / num_windows, frac_tune3 / num_windows
    return int(num_steps * f1), int(num_steps * f2), (int(num_steps * f3) if f3 != 0 else 0)


def _kernel_rule(kernel):
    """(random-generator-arg kernel?, steps_rule, min_steps) of a kernel built by this package's adjusted MCLMC."""
    if getattr(kernel, "coefficients", None) is None or not hasattr(kernel, "device_rule"):
        raise TypeError("mclmc_kernel must be a kernel built by blackjax_b200.adjusted_mclmc.build_kernel or "
                        "adjusted_mclmc_dynamic.build_kernel")
    if not getattr(kernel, "dynamic", False):
        return False, AMCLMC_STEPS_FIXED, 0
    if kernel.device_rule is None:
        raise ValueError("the tuner evaluates the default randint rule and make_random_trajectory_length_fn(...) on the "
                         "device; this integration_steps_fn has no device rule")
    rule, min_steps = kernel.device_rule
    if rule == AMCLMC_STEPS_FIXED:
        min_steps = max(int(min_steps), 1)  # make_random_trajectory_length_fn(False): max(ceil(avg), 1)
    return True, int(rule), int(min_steps)


def adjusted_mclmc_find_L_and_step_size(mclmc_kernel, logdensity_fn, num_steps, state, rng_key, target, frac_tune1=0.1,
                                        frac_tune2=0.1, frac_tune3=0.0, diagonal_preconditioning=True, params=None,
                                        max="avg", num_windows=1, tuning_factor=1.3, target_num_integration_steps=2.0, *,
                                        max_history_bytes=1 << 31):
    """blackjax/adaptation/adjusted_mclmc_adaptation.py:26-205 for every chain.

    ``mclmc_kernel`` must come from ``blackjax_b200.adjusted_mclmc.build_kernel`` (``state`` an HMCState) or
    ``adjusted_mclmc_dynamic.build_kernel`` (``state`` a DynamicHMCState) with the default randint rule or
    ``make_random_trajectory_length_fn(...)``: its integrator, divergence threshold, step rule and ``chain_offset`` are what
    the tuner runs with.  Positions are ``[C, D]``; ``state`` is not modified.  ``params`` (optional) gives the initial
    parameters; scalars and ``[D]`` metrics broadcast to every chain.  Without it ``L = sqrt(D)``,
    ``step_size = 0.2 sqrt(D)`` and ``M^-1 = 1``; either way L enters as ``target_num_integration_steps * step_size``.

    ``max_history_bytes`` bounds the position history of stage 3, which runs on slices of chains that fit it (the result
    does not depend on the slice size).

    Returns ``(state, MCLMCAdaptationState(L [C], step_size [C], inverse_mass_matrix [C, D]), num_integration_steps [C])``,
    the last the summed ``info.num_integration_steps`` of every tuning transition: float32 for the static kernel, which
    reports ``L / step_size``, int32 for the dynamic one.
    """
    if max not in ("avg", "max"):
        raise ValueError("max should be either 'max' or 'avg'")
    dynamic, rule, min_steps = _kernel_rule(mclmc_kernel)
    if dynamic != isinstance(state, DynamicHMCState):
        raise TypeError("the state must be a DynamicHMCState for adjusted_mclmc_dynamic's kernel and an HMCState for "
                        "adjusted_mclmc's")
    n1, n2, n3 = stage_lengths(num_steps, frac_tune1, frac_tune2, frac_tune3, num_windows)
    if frac_tune3 != 0 and n3 < 2:
        raise ValueError(f"stage 3 needs at least 2 transitions for the ESS, got int(num_steps * frac_tune3) = {n3}")
    q, logp, g = (t.clone() for t in state[:3])
    rga = state.random_generator_arg.clone().contiguous() if dynamic else None
    if rga is not None and (rga.dtype not in (torch.uint32, torch.int32) or tuple(rga.shape) != (q.shape[0], 2)):
        raise ValueError("random_generator_arg must be uint32 [n_chains, 2]")
    C, D = q.shape
    dev = q.device
    eng = get_engine(q, logdensity_fn, divergence_threshold=mclmc_kernel.divergence_threshold)
    if params is None:
        s = torch.sqrt(torch.tensor(float(D), dtype=torch.float32))
        params = MCLMCAdaptationState(s, s * 0.2, 1.0)
    L = _per_chain(params.L, (C,), dev)
    step_size = _per_chain(params.step_size, (C,), dev)
    imm = _per_chain(params.inverse_mass_matrix, (C, D), dev)
    count = torch.empty(C, dtype=torch.float32, device=dev)
    eng.set_integrator(mclmc_kernel.coefficients)
    # libbjx checks the configuration against the installed metric; the tuner runs with its own copy `imm`, which it
    # rewrites, so the engine's cached metric is dropped afterwards
    eng._tune_metric = imm.clone()
    eng.ensure_metric(eng._tune_metric, diagonal_only=True)
    keys = as_keys(rng_key, C, dev)
    eng._key_mode(keys, getattr(mclmc_kernel, "chain_offset", 0))
    try:
        check(lib().bjx_adjusted_mclmc_find_l_and_step_size(
            eng.h, ptr(keys), ptr(q), ptr(logp), ptr(g), ptr(rga), rule, min_steps, ptr(step_size), ptr(L), ptr(imm),
            int(num_windows), n1, n2, n3, float(target), int(bool(diagonal_preconditioning)), int(max == "max"),
            float(tuning_factor), float(target_num_integration_steps), L_FACTOR, int(max_history_bytes), ptr(count)),
            eng.h)
    finally:
        eng._imm_key = None
    final = DynamicHMCState(q, logp, g, rga) if dynamic else HMCState(q, logp, g)
    return final, MCLMCAdaptationState(L, step_size, imm), (count.to(torch.int32) if dynamic else count)


def tune_step_(eng, keys, state, step_size, L, da_state, streaming, count, mask, fix_L, target, device_rule=None,
               chain_offset=0):
    """One tuning step (dual_avg_step, :236-311) in place, libbjx ``bjx_adjusted_mclmc_tune_step``, on the engine's
    installed metric.  ``state`` = (q, logp, g) or (q, logp, g, random_generator_arg) with ``device_rule = (rule,
    min_steps)`` of the dynamic kernel; ``step_size``, ``L`` [C]; ``da_state`` [C, 5]; ``streaming`` = (total [C], moments
    [C, 2, D]) or None; ``count`` [C] or None.  All are updated in place.  Returns (success [C] bool, steps [C] int32)."""
    q, logp, g = state[:3]
    rga = state[3] if len(state) > 3 else None
    rule, min_steps = device_rule if device_rule is not None else (AMCLMC_STEPS_FIXED, 0)
    keys = as_keys(keys, eng.C, eng.device)
    eng._key_mode(keys, chain_offset)
    total, moments = streaming if streaming is not None else (None, None)
    success = torch.empty(eng.C, dtype=torch.uint8, device=eng.device)
    steps = torch.empty(eng.C, dtype=torch.int32, device=eng.device)
    check(lib().bjx_adjusted_mclmc_tune_step(eng.h, ptr(keys), ptr(q), ptr(logp), ptr(g), ptr(rga), int(rule),
                                             int(min_steps), ptr(step_size), ptr(L), ptr(da_state), ptr(total),
                                             ptr(moments), ptr(count), int(mask), int(bool(fix_L)), float(target),
                                             ptr(success), ptr(steps)), eng.h)
    return success.bool(), steps
