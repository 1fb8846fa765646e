"""ChEES-HMC warm-up: cross-chain adaptation of the step size and the trajectory length of jittered HMC.

Mirrors ``blackjax.chees_adaptation`` (blackjax/adaptation/chees_adaptation.py:574-1025) for its default configuration
(``mass_matrix_estimation=None``: identity metric, base-2 Halton jitter).  Every warm-up step is one HMC transition of all
chains with ``ceil(jitter(i) * T / eps)`` leapfrog steps followed by ``bjx_chees_update`` (libbjx): block statistics of the
proposals, two all-gathers when the chains are sharded over GPUs, dual averaging on the harmonic-mean acceptance
(:341-360) and Adam on ``log T`` along the ChEES gradient (:362-511), all on the device -- no host round trip per step.

``optim`` stands in for the reference's ``optax.adam(learning_rate, b1, b2)`` (optax is not available here): pass
``blackjax_b200.adaptation.chees_adaptation.adam(learning_rate, b1=0.9, b2=0.999)``.

``mass_matrix_estimation="diagonal"`` (:61-237,797-1001) estimates a diagonal inverse mass matrix from the positions of
all chains over the last ``mass_matrix_window_fraction`` of the warm-up, whitens the ChEES criterion by it, and floors
the trajectory length the transitions consume at (pi/2) sqrt(lambda_max), lambda_max the top eigenvalue of the whitened
ensemble covariance (``bjx_chees_update_metric``; still no host round trip per step).  The second return value is then a
:class:`ChEESMetricInfo`.
"""
import math
from typing import NamedTuple

import torch

from .. import random as bjx_random
from .._lib import CHEES_LENGTH_FLOOR, CHEES_WHITEN, check, lib, ptr
from ..base import AdaptationAlgorithm, AdaptationResults
from ..mcmc import dynamic_hmc, hmc

OPTIMAL_TARGET_ACCEPTANCE_RATE = 0.651   # chees_adaptation.py:20


class adam(NamedTuple):
    """optax.adam(learning_rate, b1, b2) (eps = 1e-8), the optimiser the reference's examples pass as ``optim``."""
    learning_rate: float
    b1: float = 0.9
    b2: float = 0.999


def halton_sequence(i: int, max_bits: int = 10) -> float:
    """blackjax/mcmc/dynamic_hmc.py:205-215."""
    return sum((((int(i) + 1) >> k) & 1) * (0.5 / (1 << k)) for k in range(int(max_bits)))


LENGTH_FLOOR_RECOMPUTE_INTERVAL = 32   # chees_adaptation.py:120


class ChEESMetricInfo(NamedTuple):
    """Second return value of ``run`` with ``mass_matrix_estimation="diagonal"``.  ``history`` [num_steps, 4]: step size,
    trajectory length, next step count and ChEES gradient per step, as without the metric; ``lambda_max`` and ``engaged``
    [num_steps]: the slow-direction eigenvalue estimate and whether the diagonal estimate is in use after step t (the
    values the transition of step t + 1 uses); ``floor_clipped_by_cap``: the final floor exceeded
    ``max_leapfrog_steps * step_size`` (raise ``max_leapfrog_steps`` to restore it)."""
    history: torch.Tensor
    lambda_max: torch.Tensor
    engaged: torch.Tensor
    floor_clipped_by_cap: bool


def chees_adaptation(logdensity_fn, num_chains: int, *, jitter_amount: float = 1.0,
                     target_acceptance_rate: float = OPTIMAL_TARGET_ACCEPTANCE_RATE, decay_rate: float = 0.5,
                     max_leapfrog_steps: int = 1000, mass_matrix_estimation=None, mass_matrix_window_fraction: float = 0.5,
                     _whiten_criterion: bool = True, _length_floor: bool = True, process_group=None):
    """``num_chains`` is the number of chains of THIS process (``positions.shape[0]``); with a ``process_group`` the
    statistics are pooled over the chains of all its ranks.  ``mass_matrix_estimation``: None (identity metric) or
    "diagonal"; ``mass_matrix_window_fraction`` in [0, 1]: the accumulation window starts at
    ``int(fraction * num_steps)`` (1.0: never, the identity metric throughout).  ``_whiten_criterion`` and
    ``_length_floor`` are the reference's private ablation switches of the diagonal mode."""
    if mass_matrix_estimation not in (None, "diagonal"):   # chees_adaptation.py:718-727
        raise ValueError(f"mass_matrix_estimation must be None or 'diagonal', got {mass_matrix_estimation!r}.")
    if not 0.0 <= mass_matrix_window_fraction <= 1.0:
        raise ValueError(f"mass_matrix_window_fraction must be in [0.0, 1.0], got {mass_matrix_window_fraction}.")
    options = 0
    if mass_matrix_estimation == "diagonal":
        options = (CHEES_WHITEN if _whiten_criterion else 0) | (CHEES_LENGTH_FLOOR if _length_floor else 0)

    def run(rng_key, positions, step_size: float, optim: adam, num_steps: int = 1000, *, max_sampling_steps: int = 1000):
        from .._comm import nccl_comm
        from .._engine import get_engine
        positions = positions.contiguous()
        C, D = positions.shape
        if C != num_chains:
            raise ValueError("initial `positions` leading dimension must be equal to the `num_chains`")
        dev = positions.device
        comm, n_ranks, rank = nccl_comm(dev, process_group)
        max_bits = int(math.ceil(math.log2(num_steps + max_sampling_steps)))
        diagonal = mass_matrix_estimation == "diagonal"
        L_ = lib()
        if diagonal:
            n_ms = L_.bjx_chees_metric_state_floats(C, D, n_ranks, options)
            if n_ms <= 0:
                raise ValueError("mass_matrix_estimation='diagonal' is built for dim <= 1024")
        kernel = hmc.build_kernel(full_info=True, chain_offset=rank * C)
        state = hmc.init(positions, logdensity_fn)
        eng = get_engine(positions, logdensity_fn)
        st = torch.empty(L_.bjx_chees_state_floats(C, D, n_ranks), dtype=torch.float32, device=dev)
        eps_c = torch.empty(C, dtype=torch.float32, device=dev)
        steps_c = torch.empty(C, dtype=torch.int32, device=dev)
        hist = torch.empty(num_steps, 4, dtype=torch.float32, device=dev)
        check(L_.bjx_chees_init(eng.h, ptr(st), float(step_size), max_bits, float(jitter_amount), ptr(eps_c), ptr(steps_c)), eng.h)
        hyper = (float(optim.learning_rate), float(optim.b1), float(optim.b2), float(target_acceptance_rate), float(decay_rate),
                 int(max_leapfrog_steps))
        if diagonal:
            ms = torch.empty(n_ms, dtype=torch.float32, device=dev)
            lam = torch.empty(num_steps, dtype=torch.float32, device=dev)
            eng_flag = torch.empty(num_steps, dtype=torch.float32, device=dev)
            imm = torch.empty(D, dtype=torch.float32, device=dev)
            check(L_.bjx_chees_metric_init(eng.h, ptr(ms), n_ranks, options, ptr(imm)), eng.h)
            # the update rewrites imm and re-installs it on the handle: the kernel's metric cache stays keyed on this tensor
            eng._imm, eng._imm_key = imm, (imm.data_ptr(), tuple(imm.shape), imm._version, str(imm.device))
            window_start = int(mass_matrix_window_fraction * num_steps)          # chees_adaptation.py:799
            floor_on = bool(options & CHEES_LENGTH_FLOOR)

            def update(t, init_q, new_q, info):
                in_window = t >= window_start
                recompute = floor_on and in_window and t % LENGTH_FLOOR_RECOMPUTE_INTERVAL == 0
                return L_.bjx_chees_update_metric(eng.h, comm, n_ranks, options, ptr(st), ptr(ms), ptr(init_q),
                                                  ptr(info.proposal.position), ptr(info.proposal.momentum), ptr(new_q),
                                                  ptr(info.acceptance_rate), ptr(info.is_divergent.to(torch.uint8)), *hyper,
                                                  int(in_window), int(recompute), ptr(eps_c), ptr(steps_c), ptr(hist), ptr(imm),
                                                  ptr(lam), ptr(eng_flag))
        else:
            imm = torch.ones(D, dtype=torch.float32, device=dev)

            def update(t, init_q, new_q, info):
                return L_.bjx_chees_update(eng.h, comm, n_ranks, ptr(st), ptr(init_q), ptr(info.proposal.position),
                                           ptr(info.proposal.momentum), ptr(info.acceptance_rate),
                                           ptr(info.is_divergent.to(torch.uint8)), *hyper, ptr(eps_c), ptr(steps_c), ptr(hist))
        keys = bjx_random.split(rng_key.to(dev), num_steps)
        for t in range(num_steps):
            init_q = state.position
            state, info = kernel(keys[t], state, logdensity_fn, eps_c, imm, steps_c)
            check(update(t, init_q, state.position, info), eng.h)
        import ctypes as C_
        out = (C_.c_float * 4)()                                             # the one host read of the warm-up
        if diagonal:
            check(L_.bjx_chees_final_metric(eng.h, comm, n_ranks, options, ptr(st), ptr(ms), int(max_leapfrog_steps), ptr(imm),
                                            out), eng.h)
            imm.add_(0.0)  # version bump: later users of imm re-derive mass_matrix_sqrt from the contents the device wrote
            eng._imm_key = (imm.data_ptr(), tuple(imm.shape), imm._version, str(imm.device))
        else:
            check(L_.bjx_chees_final(eng.h, ptr(st), out), eng.h)
        step, n_lf = float(out[0]), float(out[1])
        jitter = lambda i: halton_sequence(i, max_bits) * jitter_amount + (1.0 - jitter_amount)
        parameters = {
            "step_size": step,
            "inverse_mass_matrix": imm,
            "next_random_arg_fn": lambda i: i + 1,
            "integration_steps_fn": lambda i, n: int(math.ceil(jitter(i) * n)),
            "integration_steps_params": (n_lf,),
        }
        last = dynamic_hmc.DynamicHMCState(state.position, state.logdensity, state.logdensity_grad, num_steps)
        if diagonal:
            return AdaptationResults(last, parameters), ChEESMetricInfo(hist.cpu(), lam.cpu(), eng_flag.cpu().bool(), bool(out[2]))
        return AdaptationResults(last, parameters), hist.cpu()

    return AdaptationAlgorithm(run)
