"""The multivariate slice sampler (``blackjax.slice_sampling``, blackjax/mcmc/slice.py) behind BlackJAX's
``init / build_kernel / as_top_level_api`` surface, one fused kernel per transition: the random direction, the slice
level, the interval (Neal's doubling with its acceptance test, or stepping out) and the shrinkage, with a different
number of target evaluations on every chain.  The chain axis is explicit as in :mod:`blackjax_b200.mcmc.hmc`.

The proposal generator is :func:`direction_proposal` (``scale``: a scalar, [D], or a dense [D, D] matrix at dim
<= 128) and the interval :func:`doubling` or :func:`stepping_out`; both run on the device, so other callables raise
``NotImplementedError``.  ``width`` is a scalar or one per chain ([C]).

The device evaluates the target fewer times than the reference and decides the same.  The one deviation: the doubling
acceptance test stops after ``max_expansions + 1`` bisections and returns its verdict as it stands.  A finite bracket
never needs more; only a bracket whose width ``width * 2**j`` overflowed to inf would, and there the reference never
stops."""
from typing import NamedTuple

import numpy as np
import torch

from .._engine import get_engine
from .._lib import SLICE_DOUBLING, SLICE_STEPPING_OUT
from ..base import build_sampling_algorithm

__all__ = ["SliceState", "SliceInfo", "init", "build_kernel", "as_top_level_api", "direction_proposal", "doubling",
           "stepping_out"]


class SliceState(NamedTuple):
    """slice.py SliceState, batched: position [C,D], logdensity [C]."""

    position: torch.Tensor
    logdensity: torch.Tensor


class SliceInfo(NamedTuple):
    """slice.py SliceInfo, batched: is_accepted (bool), num_expansions, num_shrink (int32), bracket_left and
    bracket_right (float32, the bracket in t with the current point at t = 0), all [C]."""

    is_accepted: torch.Tensor
    num_expansions: torch.Tensor
    num_shrink: torch.Tensor
    bracket_left: torch.Tensor
    bracket_right: torch.Tensor


def init(position, logdensity_fn):
    """slice.py init."""
    eng = get_engine(position, logdensity_fn)
    position = position.contiguous()
    logp, _ = eng.init_state(position)  # the gradient row the targets also form is not part of this state
    return SliceState(position, logp)


def doubling(*args, **kwargs):
    """Neal (2003) Fig. 4 doubling interval with the Fig. 6 acceptance test (slice.py doubling).  Pass it as
    ``interval=doubling``; it runs inside the device kernel."""
    raise NotImplementedError("the doubling interval runs on the device: pass it as interval=doubling")


def stepping_out(*args, **kwargs):
    """Neal (2003) Fig. 3 stepping-out interval (slice.py stepping_out).  Pass it as ``interval=stepping_out``; it runs
    inside the device kernel."""
    raise NotImplementedError("the stepping-out interval runs on the device: pass it as interval=stepping_out")


def _interval_code(interval):
    if interval is None or interval is doubling:
        return SLICE_DOUBLING
    if interval is stepping_out:
        return SLICE_STEPPING_OUT
    raise NotImplementedError("slice sampling runs the doubling and stepping_out intervals of "
                              f"blackjax_b200.mcmc.slice on the device; got {interval!r}")


def _check_caps(max_expansions, max_shrinkage):
    if int(max_expansions) < 0 or int(max_shrinkage) < 0:
        raise ValueError("max_expansions and max_shrinkage must be >= 0")


def direction_proposal(scale=1.0):
    """slice.py direction_proposal: slice along the random direction ``n / |n|``, ``n = scale * z`` (a scalar or [D]
    scale) or ``scale @ z`` (a dense [D, D] scale, dim <= 128), ``z`` standard normal."""

    def proposal_generator(rng_key, position, logdensity_fn):
        raise NotImplementedError("direction_proposal runs on the device: pass it as proposal_generator to "
                                  "slice_sampling or to the kernel of build_kernel")

    proposal_generator.slice_direction_scale = scale
    return proposal_generator


def _scale_of(proposal_generator):
    scale = getattr(proposal_generator, "slice_direction_scale", None)
    if scale is None:
        raise NotImplementedError("slice sampling runs the proposal generator direction_proposal(scale) of "
                                  f"blackjax_b200.mcmc.slice on the device; got {proposal_generator!r}")
    return scale


def build_kernel(interval=doubling, max_expansions: int = 10, max_shrinkage: int = 100, inplace: bool = False,
                 chain_offset: int = 0):
    """slice.py build_kernel: ``kernel(rng_key, state, logdensity_fn, proposal_generator, width=1.0)``.
    ``inplace=True`` overwrites the input state's tensors; ``chain_offset`` is the global index of this process's first
    chain when one shared ``rng_key`` is split across GPUs."""
    code = _interval_code(interval)
    _check_caps(max_expansions, max_shrinkage)
    scales = {}  # the scale as a device tensor, converted once per device so that the engine's cache key holds

    def kernel(rng_key, state, logdensity_fn, proposal_generator, width=1.0):
        scale = _scale_of(proposal_generator)
        q, logp = state
        eng = get_engine(q, logdensity_fn)
        dev = str(eng.device)
        if isinstance(scale, torch.Tensor) or np.ndim(scale) > 0:
            key = (id(scale), dev)
            if key not in scales:
                scales[key] = (scale, torch.as_tensor(scale, dtype=torch.float32).to(eng.device))
            scale = scales[key][1]
        eng.ensure_slice_scale(scale)
        C = eng.C
        acc = torch.empty(C, dtype=torch.uint8, device=eng.device)
        n_exp = torch.empty(C, dtype=torch.int32, device=eng.device)
        n_shrink = torch.empty(C, dtype=torch.int32, device=eng.device)
        bl = torch.empty(C, dtype=torch.float32, device=eng.device)
        br = torch.empty(C, dtype=torch.float32, device=eng.device)
        out = (q, logp) if inplace else None
        qo, lo = eng.slice_step(rng_key, q, logp, width, code, max_expansions, max_shrinkage, out=out,
                                info_fields=dict(is_accepted=acc, num_expansions=n_exp, num_shrink=n_shrink,
                                                 bracket_left=bl, bracket_right=br),
                                chain_offset=chain_offset)
        return SliceState(qo, lo), SliceInfo(acc.bool(), n_exp, n_shrink, bl, br)

    return kernel


def as_top_level_api(logdensity_fn, *, proposal_generator=direction_proposal(), width=1.0, interval=doubling,
                     max_expansions: int = 10, max_shrinkage: int = 100):
    """slice.py as_top_level_api: ``blackjax.slice_sampling``."""
    _scale_of(proposal_generator)
    kernel = build_kernel(interval, max_expansions, max_shrinkage)
    return build_sampling_algorithm(kernel, init, logdensity_fn, kernel_args=(proposal_generator, width))
