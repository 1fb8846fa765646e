"""blackjax_b200 -- H100-native HMC/NUTS hot path behind BlackJAX's API.

``import blackjax_b200 as blackjax`` gives ``blackjax.hmc``, ``blackjax.nuts`` and
``blackjax.window_adaptation`` with the reference's ``init / build_kernel / __call__ ->
SamplingAlgorithm(init, step)`` surface (blackjax/__init__.py:70-80,104-112), natively batched over
chains and executed by hand-written sm_90a CUDA kernels through the C ABI in ``include/bjx.h``.
"""
import functools as _functools

from . import diagnostics, random, targets, util  # noqa: F401
from .diagnostics import effective_sample_size as ess  # noqa: F401
from .diagnostics import ess_bulk, ess_tail, rhat  # noqa: F401
from ._lib import BjxError  # noqa: F401
from .adaptation.window_adaptation import build_schedule, window_adaptation  # noqa: F401
from .adaptation.low_rank_adaptation import build_growing_window_schedule, window_adaptation_low_rank  # noqa: F401
from .adaptation.chees_adaptation import chees_adaptation  # noqa: F401
from .adaptation.meads_adaptation import meads_adaptation  # noqa: F401
from .adaptation.mclmc_adaptation import MCLMCAdaptationState, mclmc_find_L_and_step_size  # noqa: F401
from .adaptation.adjusted_mclmc_adaptation import adjusted_mclmc_find_L_and_step_size  # noqa: F401
from .base import AdaptationAlgorithm, AdaptationResults, GenerateSamplingAPI, SamplingAlgorithm  # noqa: F401
from . import mcmc  # noqa: F401
from .mcmc import hmc as _hmc
from .mcmc import nuts as _nuts
from .mcmc import dynamic_hmc as _dynamic_hmc
from .mcmc import ghmc as _ghmc
from .mcmc import mclmc as _mclmc
from .mcmc import adjusted_mclmc as _adjusted_mclmc
from .mcmc import adjusted_mclmc_dynamic as _adjusted_mclmc_dynamic
from .util import run_inference_algorithm, sample_hmc_native, sample_mclmc_native, sample_nuts_native  # noqa: F401
from .util import sample_adjusted_mclmc_native, sample_gist_native  # noqa: F401
from .util import sample_barker_native, sample_mala_native  # noqa: F401
from .util import sample_elliptical_slice_native, sample_slice_sampling_native  # noqa: F401
from .util import sample_random_walk_native  # noqa: F401
from .mcmc import elliptical_slice as _elliptical_slice
from .mcmc import slice as _slice
from .mcmc import random_walk as _random_walk
from .mcmc import barker as _barker
from .mcmc import mala as _mala
from .mcmc.composed import step_size as _gist_step_size
from .mcmc.composed import trajectory_length as _gist_trajectory_length

hmc = GenerateSamplingAPI(_hmc.as_top_level_api, _hmc.init, _hmc.build_kernel)     # blackjax/__init__.py:111
nuts = GenerateSamplingAPI(_nuts.as_top_level_api, _nuts.init, _nuts.build_kernel)  # blackjax/__init__.py:112
mhmc = GenerateSamplingAPI(                                                          # blackjax/__init__.py:145-151
    _functools.partial(_hmc.as_top_level_api, build_proposal=_hmc.multinomial_hmc_proposal),
    _hmc.init,
    _functools.partial(_hmc.build_kernel, build_proposal=_hmc.multinomial_hmc_proposal),
)
multinomial_hmc = mhmc  # backward-compatible alias (:152)
dhmc = GenerateSamplingAPI(_dynamic_hmc.as_top_level_api, _dynamic_hmc.init, _dynamic_hmc.build_kernel)  # :117
dynamic_hmc = dhmc  # backward-compatible alias (:118)
dmhmc = GenerateSamplingAPI(                                                         # blackjax/__init__.py:154-162
    _functools.partial(_dynamic_hmc.as_top_level_api, build_proposal=_hmc.multinomial_hmc_proposal),
    _dynamic_hmc.init,
    _functools.partial(_dynamic_hmc.build_kernel, build_proposal=_hmc.multinomial_hmc_proposal),
)

ghmc = GenerateSamplingAPI(_ghmc.as_top_level_api, _ghmc.init, _ghmc.build_kernel)   # blackjax/__init__.py:139
mclmc = GenerateSamplingAPI(_mclmc.as_top_level_api, _mclmc.init, _mclmc.build_kernel)  # blackjax/__init__.py:141
adjusted_mclmc = GenerateSamplingAPI(_adjusted_mclmc.as_top_level_api, _adjusted_mclmc.init,
                                     _adjusted_mclmc.build_kernel)
adjusted_mclmc_dynamic = GenerateSamplingAPI(_adjusted_mclmc_dynamic.as_top_level_api, _adjusted_mclmc_dynamic.init,
                                             _adjusted_mclmc_dynamic.build_kernel)
gist_trajectory_length = GenerateSamplingAPI(_gist_trajectory_length.as_top_level_api,  # blackjax/__init__.py:143
                                             _gist_trajectory_length.init, _gist_trajectory_length.build_kernel)
gist_step_size = GenerateSamplingAPI(_gist_step_size.as_top_level_api, _gist_step_size.init,  # blackjax/__init__.py:142
                                     _gist_step_size.build_kernel)
mala = GenerateSamplingAPI(_mala.as_top_level_api, _mala.init, _mala.build_kernel)  # blackjax/__init__.py:120
barker = GenerateSamplingAPI(_barker.as_top_level_api, _barker.init, _barker.build_kernel)  # blackjax/__init__.py:140
barker_proposal = barker  # blackjax/__init__.py:141
elliptical_slice = GenerateSamplingAPI(_elliptical_slice.as_top_level_api, _elliptical_slice.init,  # blackjax/__init__.py:134
                                       _elliptical_slice.build_kernel)
slice_sampling = GenerateSamplingAPI(_slice.as_top_level_api, _slice.init, _slice.build_kernel)  # blackjax/__init__.py:134
rmh = GenerateSamplingAPI(_random_walk.rmh_as_top_level_api, _random_walk.init, _random_walk.build_rmh)  # :113
irmh = GenerateSamplingAPI(_random_walk.irmh_as_top_level_api, _random_walk.init, _random_walk.build_irmh)  # :114-116
additive_step_random_walk = GenerateSamplingAPI(_random_walk.additive_step_random_walk, _random_walk.init,  # :125-129
                                                _random_walk.build_additive_step)
additive_step_random_walk.register_factory("normal_random_walk", _random_walk.normal_random_walk)

__version__ = "0.1.0"
