"""Elliptical slice sampling behind BlackJAX's ``init / build_kernel / as_top_level_api`` surface
(blackjax/mcmc/elliptical_slice.py), one fused kernel per transition: the momentum draw from the Gaussian prior
N(mean, cov), the slice level and the shrinking-bracket loop over the ellipse through the position and the momentum,
with a different number of likelihood evaluations on every chain.  The chain axis is explicit as in
:mod:`blackjax_b200.mcmc.hmc`.

The target passed as ``loglikelihood_fn`` is the log-likelihood alone; the prior enters through ``mean`` (scalar or
[D]) and ``cov`` ([D] variances or a dense [D, D] matrix; dense priors are built for dim <= 1024).

The one deviation from the reference is ``max_subiter`` (default 1000): a chain whose proposal is still below the slice
after ``max_subiter`` likelihood evaluations keeps its state and reports ``exhausted``, ``subiter = max_subiter``,
``theta = 0`` and ``momentum = nu``, where the reference would loop without end (a start whose log-likelihood is -inf,
for example).  For a continuous likelihood and a finite start the bracket falls below float32 resolution long before
1000 sub-iterations, so the results are the reference's whenever the cap is not reached."""
from typing import NamedTuple

import torch

from .._engine import get_engine
from ..base import build_sampling_algorithm

__all__ = ["EllipSliceState", "EllipSliceInfo", "init", "build_kernel", "as_top_level_api"]


class EllipSliceState(NamedTuple):
    """elliptical_slice.py:34-46, batched: position [C,D], logdensity [C] (the log-likelihood at position)."""

    position: torch.Tensor
    logdensity: torch.Tensor


class EllipSliceInfo(NamedTuple):
    """elliptical_slice.py:49-70, batched, plus ``exhausted`` [C] (bool): the chain reached ``max_subiter`` below the
    slice and kept its state."""

    momentum: torch.Tensor
    theta: torch.Tensor
    subiter: torch.Tensor
    exhausted: torch.Tensor


def init(position, logdensity_fn):
    """elliptical_slice.py:73-75."""
    eng = get_engine(position, logdensity_fn)
    position = position.contiguous()
    logl, _ = eng.init_state(position)  # the gradient row the targets also form is not part of this state
    return EllipSliceState(position, logl)


def _check_cov(cov_matrix):
    ndim = cov_matrix.ndim if isinstance(cov_matrix, torch.Tensor) else torch.as_tensor(cov_matrix).ndim
    if ndim not in (1, 2):  # elliptical_slice.py:94-105
        raise ValueError("The mass matrix has the wrong number of dimensions:"
                         f" expected 1 or 2, got {ndim}.")


def build_kernel(cov_matrix, mean, max_subiter: int = 1000, inplace: bool = False, chain_offset: int = 0):
    """elliptical_slice.py:78-123.  ``inplace=True`` overwrites the input state's tensors; ``chain_offset`` is the global
    index of this process's first chain when one shared ``rng_key`` is split across GPUs."""
    _check_cov(cov_matrix)
    if int(max_subiter) < 1:
        raise ValueError("max_subiter must be >= 1")
    prior = {}  # the prior as device tensors, converted once per device so that the engine's cache key holds

    def kernel(rng_key, state, logdensity_fn):
        q, logl = state
        eng = get_engine(q, logdensity_fn)
        dev = str(eng.device)
        if dev not in prior:
            prior[dev] = (torch.as_tensor(mean, dtype=torch.float32).to(eng.device),
                          torch.as_tensor(cov_matrix, dtype=torch.float32).to(eng.device))
        eng.ensure_elliptical_prior(*prior[dev])
        mom = torch.empty_like(q)
        theta = torch.empty(eng.C, dtype=torch.float32, device=eng.device)
        subiter = torch.empty(eng.C, dtype=torch.int32, device=eng.device)
        exhausted = torch.empty(eng.C, dtype=torch.uint8, device=eng.device)
        out = (q, logl) if inplace else None
        qo, lo = eng.elliptical_slice_step(rng_key, q, logl, max_subiter, out=out,
                                           info_fields=dict(momentum=mom, theta=theta, subiter=subiter,
                                                            exhausted=exhausted),
                                           chain_offset=chain_offset)
        return EllipSliceState(qo, lo), EllipSliceInfo(mom, theta, subiter, exhausted.bool())

    return kernel


def as_top_level_api(loglikelihood_fn, *, mean, cov, max_subiter: int = 1000):
    """elliptical_slice.py:126-166: ``blackjax.elliptical_slice``."""
    kernel = build_kernel(cov, mean, max_subiter)
    return build_sampling_algorithm(kernel, init, loglikelihood_fn)
