"""The GIST seam (blackjax/mcmc/composed/_seam.py): momentum draw, tuning-parameter draw, involution, one Metropolis test.

On the device the seam and both shipped instances are one kernel (``bjx_gist_step``): ``(key_momentum, key_tuning,
key_accept) = split(rng_key, 3)``, ``accept_prob = exp(min(delta + log_ratio, 0))``, the old state kept on rejection and
``energy`` the proposal's.  The reference's seam also takes arbitrary Python ``tuning_parameter_fn`` / ``apply_fn``
callables; there is no device code for those, so here the seam runs the two instances only, selected by the descriptor
their modules build (``trajectory_length.tuning`` / ``step_size.tuning``)."""
from typing import NamedTuple, Optional

import torch

from .. import integrators
from ..hmc import init as _hmc_init
from ..._engine import get_engine
from ..._lib import GIST_STEP_SIZE, GistParams
from ...base import build_sampling_algorithm

__all__ = ["GISTState", "GISTInfo", "init", "build_kernel", "as_top_level_api"]


class GISTState(NamedTuple):
    """_seam.py:61-74, batched: position [C,D], logdensity [C], logdensity_grad [C,D]."""

    position: torch.Tensor
    logdensity: torch.Tensor
    logdensity_grad: torch.Tensor


class GISTInfo(NamedTuple):
    """_seam.py:77-124."""

    momentum: Optional[torch.Tensor]
    tuning_parameter: object
    is_accepted: torch.Tensor
    is_divergent: torch.Tensor
    acceptance_rate: torch.Tensor
    energy: torch.Tensor
    num_integration_steps: torch.Tensor


class StepSizeTuningParameter(NamedTuple):
    """step_size.py:72-91: the step-size instance's tuning parameter (a, b, j)."""

    a: torch.Tensor
    b: torch.Tensor
    step_index: torch.Tensor


class Tuning(NamedTuple):
    """What the device kernel needs of one instance: its libbjx parameters and the integrator."""

    params: GistParams
    integrator: object


def init(position, logdensity_fn):
    """_seam.py:127-140: hmc.init, as a GISTState."""
    st = _hmc_init(position, logdensity_fn)
    return GISTState(*st)


def _step(rng_key, state, logdensity_fn, tuning, inverse_mass_matrix, step_size, divergence_threshold, full_info=False,
          inplace=False, chain_offset=0):
    """One transition of every chain: (new GISTState, dict of the bjx_gist_info fields)."""
    q, logp, g = state
    eng = get_engine(q, logdensity_fn, divergence_threshold=divergence_threshold)
    eng.set_integrator(integrators.as_coefficients(tuning.integrator))
    eng.ensure_metric(inverse_mass_matrix)
    C, dev = eng.C, eng.device
    f32 = lambda: torch.empty(C, dtype=torch.float32, device=dev)  # noqa: E731
    i32 = lambda: torch.empty(C, dtype=torch.int32, device=dev)    # noqa: E731
    u8 = lambda: torch.empty(C, dtype=torch.uint8, device=dev)     # noqa: E731
    fields = dict(acceptance_rate=f32(), is_accepted=u8(), is_divergent=u8(), energy=f32(), num_integration_steps=i32(),
                  forward=i32(), reverse=i32(), rejected=u8(), a=f32(), b=f32(), step_size=f32())
    if full_info:
        fields["momentum"] = torch.empty_like(q)
    out = (q, logp, g) if inplace else None
    qo, lo, go = eng.gist_step(rng_key, q, logp, g, tuning.params, step_size, out=out, info_fields=fields,
                               chain_offset=chain_offset)
    return GISTState(qo, lo, go), fields


def tuning_parameter(tuning, fields):
    """The instance's tuning parameter from the bjx_gist_info fields: L for the trajectory length (trajectory_length.py:
    313-316), StepSizeTuningParameter(a, b, j) for the step size (step_size.py:296-301)."""
    if tuning.params.instance == GIST_STEP_SIZE:
        return StepSizeTuningParameter(fields["a"], fields["b"], fields["forward"])
    return fields["num_integration_steps"]


def build_kernel(divergence_threshold: float = 1000, full_info: bool = False):
    """_seam.py:211-293.  ``tuning_parameter_fn`` is an instance descriptor (``trajectory_length.tuning(...)`` or
    ``step_size.tuning(...)``) and ``apply_fn`` must be None: the involution of each instance is part of its kernel."""

    def kernel(rng_key, state, logdensity_fn, tuning_parameter_fn, apply_fn, inverse_mass_matrix, step_size):
        if not isinstance(tuning_parameter_fn, Tuning) or apply_fn is not None:
            raise NotImplementedError("the GIST seam runs the shipped instances on the device: pass "
                                      "trajectory_length.tuning(...) or step_size.tuning(...) and apply_fn=None")
        new, f = _step(rng_key, state, logdensity_fn, tuning_parameter_fn, inverse_mass_matrix, step_size,
                       divergence_threshold, full_info)
        return new, GISTInfo(f.get("momentum"), tuning_parameter(tuning_parameter_fn, f), f["is_accepted"].bool(),
                             f["is_divergent"].bool(), f["acceptance_rate"], f["energy"], f["num_integration_steps"])

    return kernel


def as_top_level_api(logdensity_fn, inverse_mass_matrix, tuning_parameter_fn, apply_fn, *, step_size,
                     divergence_threshold: float = 1000):
    """_seam.py:296-341 (see build_kernel for what the tuning arguments may be)."""
    kernel = build_kernel(divergence_threshold)
    return build_sampling_algorithm(kernel, init, logdensity_fn,
                                    kernel_args=(tuning_parameter_fn, apply_fn, inverse_mass_matrix, step_size))
