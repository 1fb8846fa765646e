"""GIST with a self-tuning trajectory length (blackjax/mcmc/composed/trajectory_length.py), one fused kernel per
transition.  The reference caches the forward rollout (max_num_steps states per chain); here the proposal is re-integrated
from the initial state instead, which gives the same state bit for bit and keeps the memory per chain O(dim)."""
from typing import NamedTuple, Optional

import torch

from . import _seam as seam
from ..._lib import GIST_TRAJECTORY_LENGTH
from ..integrators import velocity_verlet
from ..._lib import GistParams
from ...base import build_sampling_algorithm

__all__ = ["GISTTrajectoryLengthInfo", "init", "tuning", "build_kernel", "as_top_level_api"]

init = seam.init


class GISTTrajectoryLengthInfo(NamedTuple):
    """trajectory_length.py:102-131."""

    momentum: Optional[torch.Tensor]
    tuning_parameter: torch.Tensor
    is_accepted: torch.Tensor
    is_divergent: torch.Tensor
    acceptance_rate: torch.Tensor
    energy: torch.Tensor
    num_integration_steps: torch.Tensor
    num_steps_to_uturn_forward: torch.Tensor
    num_steps_to_uturn_reverse: torch.Tensor
    is_no_return_rejected: torch.Tensor


def tuning(path_fraction: float = 0.5, max_num_steps: int = 1024, integrator=velocity_verlet):
    """The instance's parameters for the seam (the reference's tuning_parameter_fn / apply_fn pair)."""
    p = GistParams()
    p.instance = GIST_TRAJECTORY_LENGTH
    p.path_fraction = float(path_fraction)
    p.max_num_steps = int(max_num_steps)
    return seam.Tuning(p, integrator)


def build_kernel(integrator=velocity_verlet, divergence_threshold: float = 1000, path_fraction: float = 0.5,
                 max_num_steps: int = 1024, full_info: bool = False, inplace: bool = False, chain_offset: int = 0):
    """trajectory_length.py:369-443.  ``full_info`` materialises the momentum; ``inplace`` overwrites the input state."""
    t = tuning(path_fraction, max_num_steps, integrator)

    def kernel(rng_key, state, logdensity_fn, step_size, inverse_mass_matrix):
        new, f = seam._step(rng_key, state, logdensity_fn, t, inverse_mass_matrix, step_size, divergence_threshold,
                            full_info, inplace, chain_offset)
        L = f["num_integration_steps"]
        return new, GISTTrajectoryLengthInfo(f.get("momentum"), seam.tuning_parameter(t, f), f["is_accepted"].bool(),
                                             f["is_divergent"].bool(),
                                             f["acceptance_rate"], f["energy"], L, f["forward"], f["reverse"],
                                             f["rejected"].bool())

    return kernel


def as_top_level_api(logdensity_fn, inverse_mass_matrix, step_size, *, path_fraction: float = 0.5,
                     max_num_steps: int = 1024, divergence_threshold: float = 1000, integrator=velocity_verlet):
    """trajectory_length.py:446-515: ``blackjax.gist_trajectory_length``."""
    kernel = build_kernel(integrator, divergence_threshold, path_fraction, max_num_steps)
    return build_sampling_algorithm(kernel, init, logdensity_fn, kernel_args=(step_size, inverse_mass_matrix))
