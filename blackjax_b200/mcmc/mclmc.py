"""MCLMC, the microcanonical Langevin sampler, behind BlackJAX's ``init / build_kernel / as_top_level_api`` surface
(blackjax/mcmc/mclmc.py).

One transition is one step of the isokinetic integrator between two partial refreshes of the unit momentum, followed by
the reference's ``handle_high_energy`` and ``handle_nans``; all of it is one fused kernel (``k_mclmc_transition``).  The
chain axis is explicit as everywhere in this package: ``position`` is ``[n_chains, dim]``, ``rng_key`` is one raw key
``uint32[2]`` (chain c uses ``split(rng_key, n_global)[chain_offset + c]``) or per-chain keys ``uint32[C, 2]``.  ``L`` and
``step_size`` are scalars or per-chain ``[C]`` tensors.  ``inverse_mass_matrix`` is a scalar, ``[dim]``, or per-chain
``[n_chains, dim]`` (a 2-D array is always per-chain diagonal here); dense and low-rank metrics are not built.
"""
import math
from typing import NamedTuple

import torch

from .._engine import get_engine
from ..base import build_sampling_algorithm
from . import integrators
from .hmc import IntegratorState
from .integrators import isokinetic_mclachlan

__all__ = ["MCLMCInfo", "init", "build_kernel", "as_top_level_api"]


class MCLMCInfo(NamedTuple):
    """blackjax/mcmc/mclmc.py:37-52, batched over chains."""

    logdensity: torch.Tensor
    kinetic_change: torch.Tensor
    energy_change: torch.Tensor
    nonans: torch.Tensor


def init(position, logdensity_fn, rng_key):
    """blackjax/mcmc/mclmc.py:55-66: value_and_grad and a random unit momentum per chain."""
    if position.ndim != 2 or position.shape[1] < 2:
        raise ValueError("The target distribution must have more than 1 dimension for MCLMC.")
    eng = get_engine(position, logdensity_fn)
    position = position.contiguous()
    logp, grad, momentum = eng.mclmc_init(rng_key, position)
    return IntegratorState(position, momentum, logp, grad)


def metric_tensor(eng, inverse_mass_matrix):
    """The diagonal metric as installed on the engine: a scalar becomes a [dim] array (cached per engine and value, so a
    fixed scalar is installed once)."""
    if not isinstance(inverse_mass_matrix, (int, float)) and not (
            isinstance(inverse_mass_matrix, torch.Tensor) and inverse_mass_matrix.ndim == 0):
        return inverse_mass_matrix  # arrays (and the metrics libbjx rejects for MCLMC) go to the engine as they are
    value = float(inverse_mass_matrix)
    cached = getattr(eng, "_mclmc_scalar_imm", None)
    if cached is None or cached[0] != value:
        cached = (value, torch.full((eng.D,), value, dtype=torch.float32, device=eng.device))
        eng._mclmc_scalar_imm = cached
    return cached[1]


def energy_cutoff(dim, desired_energy_var_max_ratio, desired_energy_var):
    """cutoff = sqrt(ndims * eev_max_per_dim) (mclmc.py:125-141), in float32 like jnp.sqrt of the float product."""
    x = float(dim) * (float(desired_energy_var_max_ratio) * float(desired_energy_var))
    return float(torch.sqrt(torch.tensor(x, dtype=torch.float32))) if math.isfinite(x) else x


def build_kernel(integrator=isokinetic_mclachlan, desired_energy_var_max_ratio: float = math.inf,
                 desired_energy_var: float = 5e-4, inplace: bool = False, chain_offset: int = 0):
    """blackjax/mcmc/mclmc.py:69-145.  ``inplace=True`` overwrites the input state's tensors.  ``chain_offset``: global
    index of this process's first chain when one shared ``rng_key`` is split across GPUs."""
    coefficients = integrators.as_coefficients(integrator)

    def kernel(rng_key, state, logdensity_fn, inverse_mass_matrix, L, step_size):
        q, p, logp, g = state
        eng = get_engine(q, logdensity_fn)
        eng.set_integrator(coefficients)
        eng.ensure_metric(metric_tensor(eng, inverse_mass_matrix), diagonal_only=True)
        if not inplace:
            q, p, logp, g = q.clone(), p.clone(), logp.clone(), g.clone()
        C, dev = eng.C, eng.device
        fields = dict(kinetic_change=torch.empty(C, dtype=torch.float32, device=dev),
                      energy_change=torch.empty(C, dtype=torch.float32, device=dev),
                      nonans=torch.empty(C, dtype=torch.uint8, device=dev))
        eng.mclmc_step_(rng_key, q, p, logp, g, step_size, L,
                        energy_cutoff(eng.D, desired_energy_var_max_ratio, desired_energy_var), fields, chain_offset)
        info = MCLMCInfo(logp, fields["kinetic_change"], fields["energy_change"], fields["nonans"].bool())
        return IntegratorState(q, p, logp, g), info

    # what mclmc_find_L_and_step_size runs its native tuner with
    kernel.coefficients = coefficients
    kernel.desired_energy_var_max_ratio = desired_energy_var_max_ratio
    kernel.desired_energy_var = desired_energy_var
    kernel.chain_offset = chain_offset
    return kernel


def as_top_level_api(logdensity_fn, L, step_size, integrator=isokinetic_mclachlan, inverse_mass_matrix=1.0,
                     desired_energy_var_max_ratio=math.inf):
    """blackjax/mcmc/mclmc.py:148-212."""
    kernel = build_kernel(integrator=integrator, desired_energy_var_max_ratio=desired_energy_var_max_ratio)
    return build_sampling_algorithm(kernel, init, logdensity_fn, kernel_args=(inverse_mass_matrix, L, step_size),
                                    pass_rng_key_to_init=True)
