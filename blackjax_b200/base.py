"""API objects mirroring blackjax/base.py:88-113,154-206 and blackjax/__init__.py:70-80."""
from typing import Callable, NamedTuple


class SamplingAlgorithm(NamedTuple):
    """(init, step) pair, blackjax/base.py:88-113."""

    init: Callable
    step: Callable


class AdaptationAlgorithm(NamedTuple):
    run: Callable


class AdaptationResults(NamedTuple):
    """blackjax/adaptation/base.py:21-30."""

    state: object
    parameters: dict


def build_sampling_algorithm(kernel, init_fn, logdensity_fn, kernel_args=(), init_args=(), kernel_kwargs=None,
                             pass_rng_key_to_init=False):
    """blackjax/base.py:154-206: bind the static arguments, expose (init, step)."""
    kernel_kwargs = kernel_kwargs or {}

    def init(position, rng_key=None):
        if pass_rng_key_to_init:
            return init_fn(position, logdensity_fn, rng_key, *init_args)
        del rng_key
        return init_fn(position, logdensity_fn, *init_args)

    def step(rng_key, state):
        return kernel(rng_key, state, logdensity_fn, *kernel_args, **kernel_kwargs)

    return SamplingAlgorithm(init, step)


class GenerateSamplingAPI:
    """blackjax/__init__.py:70-80: callable API object exposing ``init`` and ``build_kernel``."""

    def __init__(self, differentiable, init_fn, build_kernel):
        self.differentiable = differentiable
        self.init = init_fn
        self.build_kernel = build_kernel

    def __call__(self, *args, **kwargs):
        return self.differentiable(*args, **kwargs)

    def register_factory(self, name, callable):
        """blackjax/__init__.py:79-80: expose ``callable`` as the attribute ``name`` (e.g.
        ``additive_step_random_walk.normal_random_walk``)."""
        setattr(self, name, callable)
