"""LAPS, the Late Adjusted Parallel Sampler (blackjax/adaptation/laps.py): an ensemble warm-up for many chains at once.

Every chain takes a step, one set of ensemble averages is formed over all chains, and a shared (step size, L, diagonal
metric) is updated from them before the next step.  Phase 1 is unadjusted MCLMC with an early stop on the fluctuation of
the ensemble mean; phase 2 is static adjusted MCLMC whose step size a bisection moves towards the target acceptance.
Both run natively on the device (libbjx ``bjx_laps_*``); the per-step averages are fixed-order sums, so two runs are
bit-identical.
"""
import numpy as np
import torch

from .. import random as bjr
from .._engine import get_engine
from ..mcmc import integrators
from ..mcmc.hmc import HMCState
from . import laps_burn_in as lb

__all__ = ["laps"]


def _phase_info(info, names, n):
    t = info[:n].cpu()
    return {k: t[:, i].clone() for i, k in enumerate(names)}


def laps(logdensity_fn, sample_init, ndims, num_steps1, num_steps2, num_chains, mesh, rng_key, microcanonical=True,
         alpha=1.9, save_frac=0.2, C=0.1, early_stop=True, r_end=0.01, bias_type=3, diagonal_preconditioning=True,
         integrator_coefficients=None, steps_per_sample=15, acc_prob=None, observables_for_bias=None,
         all_chains_info=None, diagnostics=True, contract=None, superchain_size=1, *, chunk=64):
    """blackjax.adaptation.laps.laps on this process's GPU.

    ``logdensity_fn`` is a target of ``blackjax_b200.targets``; ``sample_init(keys uint32 [N, 2]) -> [N, ndims]`` is called
    once with ``split(k1, N)``; ``rng_key`` is one raw key ``uint32 [2]`` on the device.  ``mesh`` must be None.
    ``chunk``: burn-in steps between two reads of the early-stop flag (the result does not depend on it).

    Returns ``(info, gradient_calls_per_step, acc_prob, final_state)``: ``info = {"phase_1": {...}, "phase_2": {...}}`` of
    float32 CPU tensors, one row per step (phase 1 trimmed to the steps run), or None without diagnostics;
    ``final_state`` an ``HMCState`` of the N chains.
    """
    if not microcanonical:
        raise ValueError("Only microcanonical mode is supported for LAPS.")
    if superchain_size != 1:
        raise ValueError("superchain_size > 1 needs splitR, which is not built")
    if all_chains_info is not None:
        raise ValueError("all_chains_info is not supported")
    if observables_for_bias is not None or contract is not None:
        raise ValueError("only the default observables_for_bias (identity) and contract (x -> 0) are supported")
    if mesh is not None:
        raise ValueError("mesh must be None: LAPS runs on this process's GPU")
    if bias_type not in (0, 1, 2, 3):
        raise ValueError("bias_type must be 0, 1, 2 or 3")
    N, D = int(num_chains), int(ndims)
    save_num = int(np.rint(np.float32(save_frac * num_steps1)))
    if save_num < 1:
        raise ValueError("save_frac * num_steps1 must round to at least 1 (the history of the early stop)")

    keys3 = bjr.split(rng_key, 3)
    key_init, key1, key2 = keys3[0], keys3[1], keys3[2]
    k1 = bjr.split(key_init, 2)[0]
    q0 = sample_init(bjr.split(k1, N))
    if not isinstance(q0, torch.Tensor) or tuple(q0.shape) != (N, D):
        raise ValueError(f"sample_init must return a [{N}, {D}] tensor (ndims does not match sample_init)")
    q0 = q0.to(rng_key.device, torch.float32).contiguous()
    eng = get_engine(q0, logdensity_fn)

    equi = bool(diagnostics) or bias_type == 2
    adap = lb.new_state(eng, save_num, equi)
    q, u, logp, g = lb.initialize(eng, q0, adap, save_num)
    eng.set_integrator(integrators.velocity_verlet)
    cfg = lb.config(save_num, alpha, C, r_end, bias_type, early_stop, equi)
    info1 = torch.full((max(int(num_steps1), 1), len(lb.BURN_IN_INFO)), float("nan"), device=eng.device) if diagnostics \
        else None
    n1 = lb.burn_in_run_(eng, key1, int(num_steps1), (q, u, logp, g), adap, cfg, info1, chunk)

    if integrator_coefficients is None:
        high = D > 200
        coef = integrators.omelyan if high else integrators.mclachlan
        target = acc_prob if acc_prob is not None else (0.9 if high else 0.7)
    else:
        coef = integrators.as_coefficients(integrator_coefficients)
        target = acc_prob if acc_prob is not None else 0.9
    gradient_calls_per_step = len(coef) // 2
    num_samples = int(num_steps2) // (gradient_calls_per_step * int(steps_per_sample))

    lb.switch_(eng, adap, diagonal_preconditioning)
    eng.set_integrator(coef)
    info2 = torch.full((max(num_samples, 1), len(lb.ADJUSTED_INFO)), float("nan"), device=eng.device) if diagnostics \
        else None
    lb.adjusted_run_(eng, key2, num_samples, (q, logp, g), adap, save_num, steps_per_sample, target, diagnostics, info2)
    final_state = HMCState(q, logp, g)
    if not diagnostics:
        return None, gradient_calls_per_step, target, final_state
    p1 = _phase_info(info1, lb.BURN_IN_INFO, n1)
    for k in ("bias", "observables", "R_avg", "R_max"):
        p1[k] = torch.zeros(n1)
    p2 = _phase_info(info2, lb.ADJUSTED_INFO, num_samples)
    p2["steps_per_sample"] = torch.full((num_samples,), int(steps_per_sample))
    for k in ("bias", "observables", "R_avg", "R_max"):
        p2[k] = torch.zeros(num_samples)
    return {"phase_1": p1, "phase_2": p2}, gradient_calls_per_step, target, final_state
