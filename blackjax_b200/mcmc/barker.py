"""Barker's proposal behind BlackJAX's ``init / build_kernel / as_top_level_api`` surface (blackjax/mcmc/barker.py), one
fused kernel per transition: the skew-symmetric proposal of one gradient evaluation and the Metropolis test.  The chain
axis is explicit as in :mod:`blackjax_b200.mcmc.hmc`.  Metrics: a diagonal inverse mass matrix [D] or one per chain
[C, D], or a dense one [D, D] for dim <= 128; ``None`` means ones."""
from typing import NamedTuple

import torch

from .._engine import get_engine
from ..base import build_sampling_algorithm

__all__ = ["BarkerState", "BarkerInfo", "init", "build_kernel", "as_top_level_api"]


class BarkerState(NamedTuple):
    """barker.py:34-48, batched: position [C,D], logdensity [C], logdensity_grad [C,D]."""

    position: torch.Tensor
    logdensity: torch.Tensor
    logdensity_grad: torch.Tensor


class BarkerInfo(NamedTuple):
    """barker.py:51-66."""

    acceptance_rate: torch.Tensor
    is_accepted: torch.Tensor
    proposal: BarkerState


def init(position, logdensity_fn):
    """barker.py:69-72."""
    eng = get_engine(position, logdensity_fn)
    position = position.contiguous()
    logp, grad = eng.init_state(position)
    return BarkerState(position, logp, grad)


def install_metric(eng, inverse_mass_matrix):
    """The metric of one transition: ``None`` is ones (barker.py:143-145)."""
    if inverse_mass_matrix is None:
        if getattr(eng, "_barker_ones", None) is None or eng._barker_ones.shape[0] != eng.D:
            eng._barker_ones = torch.ones(eng.D, dtype=torch.float32, device=eng.device)
        inverse_mass_matrix = eng._barker_ones
    eng.ensure_metric(inverse_mass_matrix)


def build_kernel(inplace: bool = False, chain_offset: int = 0):
    """barker.py:75-159.  ``inplace=True`` overwrites the input state's tensors; ``chain_offset`` is the global index of
    this process's first chain when one shared ``rng_key`` is split across GPUs."""

    def kernel(rng_key, state, logdensity_fn, step_size, inverse_mass_matrix=None):
        q, logp, g = state
        eng = get_engine(q, logdensity_fn)
        install_metric(eng, inverse_mass_matrix)
        acc_rate = torch.empty(eng.C, dtype=torch.float32, device=eng.device)
        is_acc = torch.empty(eng.C, dtype=torch.uint8, device=eng.device)
        prop = (torch.empty_like(q), torch.empty_like(logp), torch.empty_like(g))
        out = (q, logp, g) if inplace else None
        qo, lo, go = eng.barker_step(rng_key, q, logp, g, step_size, out=out,
                                     info_fields=dict(acceptance_rate=acc_rate, is_accepted=is_acc,
                                                      proposal_position=prop[0], proposal_logdensity=prop[1],
                                                      proposal_grad=prop[2]),
                                     chain_offset=chain_offset)
        return BarkerState(qo, lo, go), BarkerInfo(acc_rate, is_acc.bool(), BarkerState(*prop))

    return kernel


def as_top_level_api(logdensity_fn, step_size, inverse_mass_matrix=None):
    """barker.py:162-230: ``blackjax.barker`` (alias ``blackjax.barker_proposal``)."""
    kernel = build_kernel()
    return build_sampling_algorithm(kernel, init, logdensity_fn, kernel_args=(step_size, inverse_mass_matrix))
