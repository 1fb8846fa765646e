"""Adjusted MCLMC (MAMS) with a number of integration steps drawn anew for every transition and, batched, for every chain
(blackjax/mcmc/adjusted_mclmc_dynamic.py).  The transition is the fused adjusted MCLMC kernel with a per-chain step count
(``bjx_set_integration_steps``); ``random_generator_arg`` holds one key per chain, uint32 [n_chains, 2].

The two built-in step-count rules -- the default ``randint(key, (), 1, 10)`` and ``make_random_trajectory_length_fn(True)``
-- run on the device here, and ``util.sample_adjusted_mclmc_native`` recognises them and evaluates them inside the kernel.
"""
import math
from typing import Callable

import numpy as np
import torch

from .. import random as jr
from .._engine import get_engine
from .._lib import AMCLMC_STEPS_FIXED, AMCLMC_STEPS_RANDINT, AMCLMC_STEPS_UNIFORM
from ..base import build_sampling_algorithm
from . import adjusted_mclmc
from .adjusted_mclmc import rescale
from .dynamic_hmc import DynamicHMCState
from .hmc import HMCState
from .integrators import isokinetic_mclachlan

__all__ = ["init", "build_kernel", "as_top_level_api", "trajectory_length", "make_random_trajectory_length_fn",
           "halton_sequence"]


def init(position, logdensity_fn, random_generator_arg):
    """blackjax/mcmc/adjusted_mclmc_dynamic.py:31-51.  ``random_generator_arg`` is uint32 [n_chains, 2], or one key [2]
    that is split over the chains."""
    st = adjusted_mclmc.init(position, logdensity_fn)
    arg = random_generator_arg
    if isinstance(arg, torch.Tensor) and arg.dtype in (torch.uint32, torch.int32) and tuple(arg.shape) == (2,):
        arg = jr.split(arg.to(position.device), position.shape[0])
    return DynamicHMCState(st.position, st.logdensity, st.logdensity_grad, arg)


def _next_random_arg(keys):
    return jr.split(keys)[..., 1, :]  # jax.random.split(key)[1]   adjusted_mclmc_dynamic.py:58


def _integration_steps(keys, *params):
    return jr.randint(keys, (), 1, 10)  # jax.random.randint(key, (), 1, 10)   adjusted_mclmc_dynamic.py:55


# (bjx_adjusted_mclmc_sample steps_rule, min_steps) of the rules the native loop evaluates on the device
_integration_steps.device_rule = (AMCLMC_STEPS_RANDINT, 0)


def build_kernel(integration_steps_fn: Callable = _integration_steps, integrator=isokinetic_mclachlan,
                 divergence_threshold: float = 1000, next_random_arg_fn: Callable = _next_random_arg, **kw):
    """blackjax/mcmc/adjusted_mclmc_dynamic.py:54-129.  ``integration_steps_fn(random_generator_arg, *params)`` returns
    an int32 tensor [n_chains] (or an int); ``next_random_arg_fn`` maps ``random_generator_arg`` to the next one.
    ``kw`` (full_info, inplace, chain_offset) as ``adjusted_mclmc.build_kernel``."""
    static = adjusted_mclmc.build_kernel(integrator, divergence_threshold, **kw)
    device_rule = getattr(integration_steps_fn, "device_rule", None)

    def kernel(rng_key, state, logdensity_fn, step_size, L_proposal_factor=math.inf, inverse_mass_matrix=1.0,
               integration_steps_params=()):
        if device_rule is not None and device_rule[0] != AMCLMC_STEPS_RANDINT and _per_chain(integration_steps_params):
            # a per-chain average trajectory length (the tuner's L / step_size): the rule runs on the device
            eng = get_engine(state.position, logdensity_fn, divergence_threshold=divergence_threshold)
            num_integration_steps = eng.adjusted_mclmc_num_steps(device_rule, integration_steps_params[0],
                                                                 state.random_generator_arg)
        else:
            num_integration_steps = integration_steps_fn(state.random_generator_arg, *integration_steps_params)
        st = HMCState(state.position, state.logdensity, state.logdensity_grad)
        new, info = static(rng_key, st, logdensity_fn, step_size, (num_integration_steps,), inverse_mass_matrix,
                           L_proposal_factor)
        next_arg = next_random_arg_fn(state.random_generator_arg)
        return DynamicHMCState(new.position, new.logdensity, new.logdensity_grad, next_arg), info

    kernel.coefficients = static.coefficients
    kernel.divergence_threshold = divergence_threshold
    kernel.chain_offset = static.chain_offset
    kernel.device_rule = device_rule
    kernel.dynamic = True
    return kernel


def _per_chain(integration_steps_params):
    return (len(integration_steps_params) == 1 and isinstance(integration_steps_params[0], torch.Tensor)
            and integration_steps_params[0].ndim >= 1)


def as_top_level_api(logdensity_fn, step_size, L_proposal_factor=math.inf, inverse_mass_matrix=1.0, *,
                     divergence_threshold: int = 1000, integrator=isokinetic_mclachlan,
                     next_random_arg_fn: Callable = _next_random_arg, integration_steps_fn: Callable = _integration_steps,
                     integration_steps_params=(), **kw):
    """blackjax/mcmc/adjusted_mclmc_dynamic.py:132-194."""
    kernel = build_kernel(integration_steps_fn=integration_steps_fn, integrator=integrator,
                          next_random_arg_fn=next_random_arg_fn, divergence_threshold=divergence_threshold, **kw)
    return build_sampling_algorithm(kernel, init, logdensity_fn,
                                    kernel_args=(step_size, L_proposal_factor, inverse_mass_matrix,
                                                 integration_steps_params),
                                    pass_rng_key_to_init=True)


def halton_sequence(i, max_bits: int = 10):
    """blackjax/mcmc/dynamic_hmc.py:205-215: the (i+1)-th element of the base-2 Halton sequence, float32; ``i`` an int, a
    numpy integer array or an integer tensor."""
    if isinstance(i, torch.Tensor):
        b = 2 ** torch.arange(max_bits, dtype=i.dtype, device=i.device)
        bits = torch.remainder(torch.div(i[..., None] + 1, b, rounding_mode="floor"), 2).to(torch.float32)
        return (bits * (0.5 / b.to(torch.float32))).sum(-1)
    i = np.asarray(i, np.int64)
    b = 2 ** np.arange(max_bits, dtype=np.int64)
    bits = np.mod((i[..., None] + 1) // b, 2).astype(np.float32)
    return (bits * (np.float32(0.5) / b.astype(np.float32))).sum(-1, dtype=np.float32)


def trajectory_length(t, mu):
    """blackjax/mcmc/adjusted_mclmc_dynamic.py:197-212: rint(0.5 + halton(t) * rescale(mu)), int32."""
    s = rescale(mu)
    h = halton_sequence(t)
    if isinstance(h, torch.Tensor):
        return torch.round(0.5 + h * torch.tensor(s, device=h.device)).to(torch.int32)
    return np.rint(np.float32(0.5) + h * s).astype(np.int32)


def make_random_trajectory_length_fn(random_trajectory_length: bool, *, min_steps: int = 1) -> Callable:
    """blackjax/mcmc/adjusted_mclmc_dynamic.py:215-247: ``(random_generator_arg, avg_num_integration_steps) -> int32``.
    Random: ``max(ceil(uniform(key) * rescale(avg)), min_steps)`` per chain (the reference clips at 1; ``min_steps=0`` is
    the unclipped rule of its own sampling tests).  Otherwise ``max(ceil(avg), 1)`` for every chain.  A per-chain ``avg``
    tensor [C] (the tuner's ``L / step_size``) is evaluated on the device by the kernels that take this rule."""
    if random_trajectory_length:
        def integration_steps_fn(key, avg_num_integration_steps):
            u = jr.uniform(key)
            n = torch.ceil(u * torch.tensor(rescale(avg_num_integration_steps), device=u.device)).to(torch.int32)
            return torch.clamp(n, min=min_steps)

        integration_steps_fn.device_rule = (AMCLMC_STEPS_UNIFORM, int(min_steps))
    else:
        def integration_steps_fn(key, avg_num_integration_steps):
            return max(int(math.ceil(np.float32(avg_num_integration_steps))), 1)

        integration_steps_fn.device_rule = (AMCLMC_STEPS_FIXED, 0)
    return integration_steps_fn
