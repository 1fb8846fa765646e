"""Adjusted MCLMC (MAMS), the Metropolis-adjusted microcanonical sampler, behind BlackJAX's ``init / build_kernel /
as_top_level_api`` surface (blackjax/mcmc/adjusted_mclmc.py).

One transition draws a fresh unit momentum, runs ``num_integration_steps`` steps of the isokinetic integrator (each between
two partial momentum refreshes when ``L_proposal_factor`` is finite) and accepts or rejects the end state with
Metropolis-Hastings; all of it is one fused kernel (``k_amclmc_transition``).  The chain axis is explicit as everywhere in
this package: ``position`` is ``[n_chains, dim]``, ``rng_key`` is one raw key ``uint32[2]`` (chain c uses
``split(rng_key, n_global)[chain_offset + c]``) or per-chain keys ``uint32[C, 2]``.  ``step_size`` is a scalar or a per-chain
``[C]`` tensor; ``inverse_mass_matrix`` is a scalar, ``[dim]`` or per-chain ``[n_chains, dim]`` (a 2-D array is always
per-chain diagonal here); dense and low-rank metrics are not built.
"""
import math
import warnings

import numpy as np
import torch

from .._engine import get_engine
from ..base import build_sampling_algorithm
from . import hmc, integrators
from .hmc import HMCInfo, HMCState, IntegratorState
from .integrators import isokinetic_mclachlan
from .mclmc import metric_tensor

__all__ = ["init", "build_kernel", "as_top_level_api", "rescale"]


def init(position, logdensity_fn):
    """blackjax/mcmc/adjusted_mclmc.py:35-50: value_and_grad of the log-density."""
    return hmc.init(position, logdensity_fn)


def steps_argument(num_integration_steps):
    """The step count as the kernel takes it: an int, or a tensor [C] for per-chain counts.  A non-integer scalar runs
    ceil(n) steps, as the reference's ``fori_loop(0, n, ...)`` does with a float bound; so does a floating-point tensor
    (e.g. the tuner's ``L / step_size``), chain by chain on the device."""
    if isinstance(num_integration_steps, torch.Tensor) and num_integration_steps.ndim >= 1:
        return num_integration_steps
    n = float(num_integration_steps)
    if not n >= 0:
        raise ValueError("num_integration_steps must be >= 0")
    return int(math.ceil(n))


def build_kernel(integrator=isokinetic_mclachlan, divergence_threshold: float = 1000, full_info: bool = False,
                 inplace: bool = False, chain_offset: int = 0):
    """blackjax/mcmc/adjusted_mclmc.py:53-114.  ``full_info=True`` also fills ``HMCInfo.momentum`` and ``proposal``
    (D-sized).  ``inplace=True`` overwrites the input state's tensors.  ``chain_offset``: global index of this process's
    first chain when one shared ``rng_key`` is split across GPUs."""
    coefficients = integrators.as_coefficients(integrator)

    def kernel(rng_key, state, logdensity_fn, step_size, integration_steps_params=(1,), inverse_mass_matrix=1.0,
               L_proposal_factor=math.inf):
        (num_integration_steps,) = integration_steps_params
        n = steps_argument(num_integration_steps)
        q, logp, g = state
        eng = get_engine(q, logdensity_fn, divergence_threshold=divergence_threshold)
        eng.set_integrator(coefficients)
        eng.ensure_metric(metric_tensor(eng, inverse_mass_matrix), diagonal_only=True)
        C, dev = eng.C, eng.device
        fields = dict(acceptance_rate=torch.empty(C, dtype=torch.float32, device=dev),
                      is_accepted=torch.empty(C, dtype=torch.uint8, device=dev),
                      is_divergent=torch.empty(C, dtype=torch.uint8, device=dev),
                      energy=torch.empty(C, dtype=torch.float32, device=dev))
        if full_info:
            fields.update(momentum=torch.empty_like(q), proposal_position=torch.empty_like(q),
                          proposal_momentum=torch.empty_like(q))
        out = (q, logp, g) if inplace else None
        qo, lo, go = eng.adjusted_mclmc_step(rng_key, q, logp, g, step_size, n, L_proposal_factor, out=out,
                                             info_fields=fields, chain_offset=chain_offset)
        proposal = None
        if full_info:
            proposal = IntegratorState(fields["proposal_position"], fields["proposal_momentum"], None, None)
        info = HMCInfo(fields.get("momentum"), fields["acceptance_rate"], fields["is_accepted"].bool(),
                       fields["is_divergent"].bool(), fields["energy"], proposal, num_integration_steps)
        return HMCState(qo, lo, go), info

    # what adjusted_mclmc_find_L_and_step_size reads: the kernel's integrator, divergence threshold, chain offset and step
    # rule (None: the static kernel, ceil(L / step_size) steps)
    kernel.coefficients = coefficients
    kernel.divergence_threshold = divergence_threshold
    kernel.chain_offset = chain_offset
    kernel.device_rule = None
    return kernel


def as_top_level_api(logdensity_fn, step_size, L_proposal_factor=math.inf, inverse_mass_matrix=1.0, *,
                     divergence_threshold: int = 1000, integrator=isokinetic_mclachlan, num_integration_steps=None,
                     integration_steps_params=None, **kw):
    """blackjax/mcmc/adjusted_mclmc.py:117-191, with its deprecation of ``num_integration_steps``."""
    if integration_steps_params is not None and num_integration_steps is not None:
        warnings.warn(
            "Both `num_integration_steps` and `integration_steps_params` were "
            "provided. `num_integration_steps` is deprecated; "
            "`integration_steps_params` will be used.",
            DeprecationWarning,
            stacklevel=2,
        )
    if integration_steps_params is None:
        if num_integration_steps is None:
            raise ValueError("Either `num_integration_steps` or `integration_steps_params` must be provided.")
        integration_steps_params = (num_integration_steps,)
    kernel = build_kernel(integrator=integrator, divergence_threshold=divergence_threshold, **kw)
    return build_sampling_algorithm(kernel, init, logdensity_fn,
                                    kernel_args=(step_size, integration_steps_params, inverse_mass_matrix,
                                                 L_proposal_factor))


def rescale(mu):
    """blackjax/mcmc/adjusted_mclmc.py:281-288, in float32: s such that round(U(0, 1) * s + 0.5) has expected value mu."""
    F = np.float32
    mu = F(mu)
    k = np.floor(F(2) * mu - F(1))
    x = k * (mu - F(0.5) * (k + F(1))) / (k + F(1) - mu)
    return F(k + x)
