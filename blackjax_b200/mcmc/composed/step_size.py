"""GIST with a self-tuning step size (blackjax/mcmc/composed/step_size.py), one fused kernel per transition: the
doubling / halving search, the proposal at initial_step_size * 2^j and the reversibility re-search all run on the device."""
from typing import NamedTuple, Optional

import torch

from . import _seam as seam
from ._seam import StepSizeTuningParameter
from ..._lib import GIST_ASYMMETRIC, GIST_STEP_SIZE, GIST_SYMMETRIC
from ..integrators import velocity_verlet
from ..._lib import GistParams
from ...base import build_sampling_algorithm

__all__ = ["GISTStepSizeInfo", "StepSizeTuningParameter", "init", "tuning", "build_kernel", "as_top_level_api"]

init = seam.init


class GISTStepSizeInfo(NamedTuple):
    """step_size.py:104-139."""

    momentum: Optional[torch.Tensor]
    tuning_parameter: StepSizeTuningParameter
    is_accepted: torch.Tensor
    is_divergent: torch.Tensor
    acceptance_rate: torch.Tensor
    energy: torch.Tensor
    num_integration_steps: torch.Tensor
    step_index: torch.Tensor
    reverse_step_index: torch.Tensor
    search_exhausted: torch.Tensor
    step_size: torch.Tensor


def _criterion(criterion):
    if criterion not in ("symmetric", "asymmetric"):
        raise ValueError(f"criterion must be 'symmetric' or 'asymmetric', got {criterion!r}")
    return GIST_SYMMETRIC if criterion == "symmetric" else GIST_ASYMMETRIC


def tuning(num_integration_steps: int = 1, criterion: str = "symmetric", max_search_steps: int = 10,
           integrator=velocity_verlet):
    """The instance's parameters for the seam (the reference's step_size_selector and apply_fn)."""
    p = GistParams()
    p.instance = GIST_STEP_SIZE
    p.num_integration_steps = int(num_integration_steps)
    p.max_search_steps = int(max_search_steps)
    p.criterion = _criterion(criterion)
    return seam.Tuning(p, integrator)


def build_kernel(integrator=velocity_verlet, divergence_threshold: float = 1000, criterion: str = "symmetric",
                 max_search_steps: int = 10, full_info: bool = False, inplace: bool = False, chain_offset: int = 0):
    """step_size.py:349-434 (ValueError on an unknown criterion).  ``full_info`` materialises the momentum; ``inplace``
    overwrites the input state."""
    _criterion(criterion)

    def kernel(rng_key, state, logdensity_fn, initial_step_size, inverse_mass_matrix, num_integration_steps=1):
        t = tuning(num_integration_steps, criterion, max_search_steps, integrator)
        new, f = seam._step(rng_key, state, logdensity_fn, t, inverse_mass_matrix, initial_step_size,
                            divergence_threshold, full_info, inplace, chain_offset)
        tp = seam.tuning_parameter(t, f)
        return new, GISTStepSizeInfo(f.get("momentum"), tp, f["is_accepted"].bool(), f["is_divergent"].bool(),
                                     f["acceptance_rate"], f["energy"], f["num_integration_steps"], f["forward"],
                                     f["reverse"], f["rejected"].bool(), f["step_size"])

    return kernel


def as_top_level_api(logdensity_fn, inverse_mass_matrix, initial_step_size, num_integration_steps: int = 1, *,
                     criterion: str = "symmetric", max_search_steps: int = 10, divergence_threshold: float = 1000,
                     integrator=velocity_verlet):
    """step_size.py:437-509: ``blackjax.gist_step_size``."""
    kernel = build_kernel(integrator, divergence_threshold, criterion, max_search_steps)
    return build_sampling_algorithm(kernel, init, logdensity_fn,
                                    kernel_args=(initial_step_size, inverse_mass_matrix, num_integration_steps))
