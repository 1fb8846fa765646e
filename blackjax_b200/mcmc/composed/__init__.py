"""The GIST (Gibbs self-tuning) samplers (blackjax/mcmc/composed): the seam and its two instances, the self-tuning
trajectory length (``blackjax.gist_trajectory_length``) and the self-tuning step size (``blackjax.gist_step_size``), each
one fused sm_90a kernel per transition."""
from . import step_size, trajectory_length  # noqa: F401
from ._seam import GISTInfo, GISTState, build_kernel, init  # noqa: F401

__all__ = ["GISTState", "GISTInfo", "init", "build_kernel", "step_size", "trajectory_length"]
