"""NUTS behind BlackJAX's surface (blackjax/mcmc/nuts.py): iterative tree doubling driven from host
C++ (libbjx ``bjx_nuts_step``), every leapfrog leaf and the per-chain energy / U-turn reductions as
sm_90a kernels.  See :mod:`blackjax_b200.mcmc.hmc` for the batched-surface conventions."""
from typing import NamedTuple, Optional

import torch

from .._engine import get_engine
from ..base import build_sampling_algorithm
from . import hmc, integrators
from .hmc import HMCState, IntegratorState
from .integrators import velocity_verlet

__all__ = ["NUTSInfo", "init", "build_kernel", "as_top_level_api"]

init = hmc.init  # blackjax/mcmc/nuts.py:33


class NUTSInfo(NamedTuple):
    """blackjax/mcmc/nuts.py:36-74 (D-sized fields only with ``full_info=True``)."""

    momentum: Optional[torch.Tensor]
    is_divergent: torch.Tensor
    is_turning: torch.Tensor
    energy: torch.Tensor
    trajectory_leftmost_state: Optional[IntegratorState]
    trajectory_rightmost_state: Optional[IntegratorState]
    num_trajectory_expansions: torch.Tensor
    num_integration_steps: torch.Tensor
    acceptance_rate: torch.Tensor


def build_kernel(integrator=velocity_verlet, divergence_threshold: int = 1000, full_info: bool = False,
                 inplace: bool = False, max_tree_depth: int = 10, chain_offset: int = 0):
    """blackjax/mcmc/nuts.py:77-147.  ``max_tree_depth`` sizes the checkpoint workspace (upper bound for
    ``max_num_doublings``)."""
    coefficients = integrators.as_coefficients(integrator)

    def kernel(rng_key, state, logdensity_fn, step_size, inverse_mass_matrix, max_num_doublings: int = 10,
               _momentum=None, _key_integrator=None):
        q, logp, g = state
        eng = get_engine(q, logdensity_fn, max_tree_depth=max(max_tree_depth, max_num_doublings),
                         divergence_threshold=divergence_threshold)
        eng.set_integrator(coefficients)
        eng.ensure_metric(inverse_mass_matrix)
        keys = None if _key_integrator is not None else rng_key
        C, dev = eng.C, eng.device
        fields = dict(acceptance_rate=torch.empty(C, dtype=torch.float32, device=dev),
                      is_divergent=torch.empty(C, dtype=torch.uint8, device=dev),
                      is_turning=torch.empty(C, dtype=torch.uint8, device=dev),
                      energy=torch.empty(C, dtype=torch.float32, device=dev),
                      num_integration_steps=torch.empty(C, dtype=torch.int32, device=dev),
                      num_trajectory_expansions=torch.empty(C, dtype=torch.int32, device=dev))
        if full_info:
            for k in ("momentum", "left_position", "left_momentum", "right_position", "right_momentum"):
                fields[k] = torch.empty_like(q)
        out = (q, logp, g) if inplace else None
        qo, lo, go = eng.nuts_step(keys, q, logp, g, step_size, max_num_doublings, out=out, info_fields=fields,
                                   momentum=_momentum, key_integrator=_key_integrator, chain_offset=chain_offset)
        left = right = None
        if full_info:
            left = IntegratorState(fields["left_position"], fields["left_momentum"], None, None)
            right = IntegratorState(fields["right_position"], fields["right_momentum"], None, None)
        info = NUTSInfo(fields.get("momentum"), fields["is_divergent"].bool(), fields["is_turning"].bool(),
                        fields["energy"], left, right, fields["num_trajectory_expansions"],
                        fields["num_integration_steps"], fields["acceptance_rate"])
        return HMCState(qo, lo, go), info

    return kernel


def as_top_level_api(logdensity_fn, step_size, inverse_mass_matrix, *, max_num_doublings: int = 10,
                     divergence_threshold: int = 1000, integrator=velocity_verlet, **kw):
    """blackjax/mcmc/nuts.py:150-220."""
    kernel = build_kernel(integrator, divergence_threshold, max_tree_depth=max_num_doublings, **kw)
    return build_sampling_algorithm(kernel, init, logdensity_fn,
                                    kernel_args=(step_size, inverse_mass_matrix, max_num_doublings))
