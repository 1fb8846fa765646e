"""MALA behind BlackJAX's ``init / build_kernel / as_top_level_api`` surface (blackjax/mcmc/mala.py), one fused kernel per
transition: the Euler step of the overdamped Langevin diffusion, one gradient evaluation and the Metropolis test with
the asymmetric transition energies.  The chain axis is explicit as in :mod:`blackjax_b200.mcmc.hmc`."""
from typing import NamedTuple

import torch

from .._engine import get_engine
from ..base import build_sampling_algorithm

__all__ = ["MALAState", "MALAInfo", "init", "build_kernel", "as_top_level_api"]


class MALAState(NamedTuple):
    """mala.py:30-41, batched: position [C,D], logdensity [C], logdensity_grad [C,D]."""

    position: torch.Tensor
    logdensity: torch.Tensor
    logdensity_grad: torch.Tensor


class MALAInfo(NamedTuple):
    """mala.py:44-57."""

    acceptance_rate: torch.Tensor
    is_accepted: torch.Tensor


def init(position, logdensity_fn):
    """mala.py:60-63."""
    eng = get_engine(position, logdensity_fn)
    position = position.contiguous()
    logp, grad = eng.init_state(position)
    return MALAState(position, logp, grad)


def build_kernel(inplace: bool = False, chain_offset: int = 0):
    """mala.py:66-117.  ``inplace=True`` overwrites the input state's tensors; ``chain_offset`` is the global index of
    this process's first chain when one shared ``rng_key`` is split across GPUs."""

    def kernel(rng_key, state, logdensity_fn, step_size):
        q, logp, g = state
        eng = get_engine(q, logdensity_fn)
        acc_rate = torch.empty(eng.C, dtype=torch.float32, device=eng.device)
        is_acc = torch.empty(eng.C, dtype=torch.uint8, device=eng.device)
        out = (q, logp, g) if inplace else None
        qo, lo, go = eng.mala_step(rng_key, q, logp, g, step_size, out=out,
                                   info_fields=dict(acceptance_rate=acc_rate, is_accepted=is_acc),
                                   chain_offset=chain_offset)
        return MALAState(qo, lo, go), MALAInfo(acc_rate, is_acc.bool())

    return kernel


def as_top_level_api(logdensity_fn, step_size):
    """mala.py:120-172: ``blackjax.mala``."""
    kernel = build_kernel()
    return build_sampling_algorithm(kernel, init, logdensity_fn, kernel_args=(step_size,))
