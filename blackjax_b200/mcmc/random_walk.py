"""Random-walk Rosenbluth-Metropolis-Hastings (blackjax/mcmc/random_walk.py: ``additive_step_random_walk``,
``normal_random_walk``, ``rmh``, ``irmh``) behind BlackJAX's ``init / build_kernel / as_top_level_api`` surface, one
fused kernel per transition: the Gaussian proposal, one target evaluation and the accept decision.  The chain axis is
explicit as in :mod:`blackjax_b200.mcmc.hmc`.

Callables cannot run on the device, so the proposal generators are descriptors, as ``slice.direction_proposal`` is:

* :func:`normal` ``(sigma)``: the additive step ``x + sigma z`` (``build_additive_step``, ``normal_random_walk``);
* :func:`gaussian_proposal` ``(sigma, mean=None)``: rmh's transition generator, ``x + sigma z`` without a mean and the
  position-independent ``mean + sigma z`` with one;
* :func:`gaussian_distribution` ``(mean, sigma)``: irmh's ``proposal_distribution``, ``mean + sigma z``;
* :func:`gaussian_logdensity` ``(mean, sigma)``: the ``proposal_logdensity_fn`` of a position-independent proposal of the
  same ``mean`` and ``sigma``, ``log N(x; mean, diag(sigma)^2)`` without its constant terms (they cancel).

``sigma`` is a scalar, [D], or a dense [D, D] matrix at dim <= 128 (``sigma @ z``); ``gaussian_logdensity`` takes a
scalar or [D] sigma.  Any other callable raises ``NotImplementedError``.

As in the reference, the state's stored ``logdensity`` is used as given, never re-evaluated, and
``RWInfo.proposal`` holds the state *after* the accept decision (random_walk.py:398-399), not the candidate."""
from typing import NamedTuple

import numpy as np
import torch

from .._engine import get_engine
from .._lib import RW_ADDITIVE, RW_INDEPENDENT
from ..base import build_sampling_algorithm

__all__ = ["RWState", "RWInfo", "init", "normal", "gaussian_proposal", "gaussian_distribution", "gaussian_logdensity",
           "build_additive_step", "additive_step_random_walk", "normal_random_walk", "build_irmh",
           "irmh_as_top_level_api", "build_rmh", "rmh_as_top_level_api"]

_DESCRIPTORS = ("normal, gaussian_proposal, gaussian_distribution and gaussian_logdensity of "
                "blackjax_b200.mcmc.random_walk")


class RWState(NamedTuple):
    """random_walk.py RWState, batched: position [C,D], logdensity [C]."""

    position: torch.Tensor
    logdensity: torch.Tensor


class RWInfo(NamedTuple):
    """random_walk.py RWInfo, batched: acceptance_rate (float32 [C]), is_accepted (bool [C]) and proposal, which, as in
    the reference, is the state after the accept decision (the new state), not the candidate."""

    acceptance_rate: torch.Tensor
    is_accepted: torch.Tensor
    proposal: RWState


def init(position, logdensity_fn):
    """random_walk.py init."""
    eng = get_engine(position, logdensity_fn)
    position = position.contiguous()
    logp, _ = eng.init_state(position)  # the gradient row the targets also form is not part of this state
    return RWState(position, logp)


def _check_sigma(sigma):
    if np.ndim(sigma) > 2:
        raise ValueError("sigma must be a vector or a matrix.")


def normal(sigma):
    """random_walk.py normal: the additive step ``sigma * z`` ([D] or scalar sigma) or ``sigma @ z`` ([D, D], dim
    <= 128), ``z`` standard normal.  Pass it as ``random_step``; it runs inside the device kernel."""
    _check_sigma(sigma)

    def propose(rng_key, position):
        raise NotImplementedError("normal(sigma) runs on the device: pass it as random_step to "
                                  "additive_step_random_walk or to the kernel of build_additive_step")

    propose.rw_proposal = (RW_ADDITIVE, sigma, None)
    propose.rw_role = "random_step"
    return propose


def gaussian_proposal(sigma, mean=None):
    """rmh's transition generator: ``position + sigma z`` (``mean=None``) or the position-independent ``mean + sigma z``,
    with ``sigma`` as in :func:`normal`.  Pass it as ``proposal_generator``; it runs inside the device kernel."""
    _check_sigma(sigma)

    def transition_generator(rng_key, position):
        raise NotImplementedError("gaussian_proposal runs on the device: pass it as the transition generator of rmh")

    transition_generator.rw_proposal = (RW_ADDITIVE, sigma, None) if mean is None else (RW_INDEPENDENT, sigma, mean)
    transition_generator.rw_role = "transition_generator"
    return transition_generator


def gaussian_distribution(mean, sigma):
    """irmh's ``proposal_distribution``: ``mean + sigma z``, independent of the position, with ``sigma`` as in
    :func:`normal`.  It runs inside the device kernel."""
    _check_sigma(sigma)

    def proposal_distribution(rng_key):
        raise NotImplementedError("gaussian_distribution runs on the device: pass it as the proposal_distribution of "
                                  "irmh")

    proposal_distribution.rw_proposal = (RW_INDEPENDENT, sigma, mean)
    proposal_distribution.rw_role = "proposal_distribution"
    return proposal_distribution


def gaussian_logdensity(mean, sigma):
    """The ``proposal_logdensity_fn`` of the position-independent Gaussian proposal N(mean, diag(sigma)^2) (scalar or
    [D] sigma): ``f(new_state, prev_state) = -0.5 sum ((prev_state.position - mean) / sigma)^2``, the log-density of the
    proposal that reaches the previous position, without the constant terms that cancel in the acceptance ratio.  rmh
    and irmh accept it only with a position-independent proposal of the same ``mean`` and ``sigma``."""
    if np.ndim(sigma) > 1:
        raise ValueError("gaussian_logdensity takes a scalar or [D] sigma: a dense sigma is not built")

    def proposal_logdensity_fn(new_state, prev_state):
        raise NotImplementedError("gaussian_logdensity runs on the device: pass it as the proposal_logdensity_fn of "
                                  "rmh or irmh")

    proposal_logdensity_fn.rw_correction = (mean, sigma)
    return proposal_logdensity_fn


_ROLES = {"random_step": "normal(sigma)", "transition_generator": "gaussian_proposal(sigma, mean=None)",
          "proposal_distribution": "gaussian_distribution(mean, sigma)"}


def _proposal_of(fn, role):
    """The (kind, sigma, mean) of a proposal descriptor in the role the kernel gives it."""
    desc = getattr(fn, "rw_proposal", None)
    if desc is None:
        raise NotImplementedError(f"random-walk Metropolis runs the descriptors {_DESCRIPTORS} on the device; got "
                                  f"{fn!r} as {role}")
    if fn.rw_role != role:
        raise ValueError(f"{role} must be {_ROLES[role]}, got the {fn.rw_role} {_ROLES[fn.rw_role]}")
    return desc


def _same(a, b):
    if a is b:
        return True
    if isinstance(a, torch.Tensor) or isinstance(b, torch.Tensor):
        a, b = (t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else t for t in (a, b))
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and bool(np.array_equal(a, b))


def _correct_of(desc, proposal_logdensity_fn):
    """Whether the correction applies (False for None); raises unless it pairs with a position-independent proposal of
    the same mean and sigma."""
    if proposal_logdensity_fn is None:
        return False
    corr = getattr(proposal_logdensity_fn, "rw_correction", None)
    if corr is None:
        raise NotImplementedError(f"random-walk Metropolis runs the descriptors {_DESCRIPTORS} on the device; got "
                                  f"{proposal_logdensity_fn!r} as proposal_logdensity_fn")
    kind, sigma, mean = desc
    if kind != RW_INDEPENDENT or not (_same(corr[0], mean) and _same(corr[1], sigma)):
        raise ValueError("gaussian_logdensity(mean, sigma) corrects only the position-independent proposal of the same "
                         "mean and sigma (gaussian_distribution(mean, sigma) or gaussian_proposal(sigma, mean))")
    return True


class _Runner:
    """What the three kernels share: the descriptors' arrays as device tensors (converted once per device, so that the
    engine's cache key holds), the verdict of each (proposal, correction) pairing, and the transition itself."""

    def __init__(self, inplace, chain_offset):
        self.inplace, self.chain_offset = inplace, chain_offset
        self.arrays, self.pairs = {}, {}

    def _dev(self, a, dev):
        if a is None or not (isinstance(a, torch.Tensor) or np.ndim(a) > 0):
            return a
        key = (id(a), str(dev))
        if key not in self.arrays:
            self.arrays[key] = (a, torch.as_tensor(a, dtype=torch.float32).to(dev))
        return self.arrays[key][1]

    def correct(self, fn, proposal_logdensity_fn):
        if proposal_logdensity_fn is None:
            return False
        key = (id(fn), id(proposal_logdensity_fn))
        if key not in self.pairs:
            self.pairs[key] = (fn, proposal_logdensity_fn, _correct_of(fn.rw_proposal, proposal_logdensity_fn))
        return self.pairs[key][2]

    def __call__(self, rng_key, state, logdensity_fn, fn, role, proposal_logdensity_fn=None):
        kind, sigma, mean = _proposal_of(fn, role)
        correct = self.correct(fn, proposal_logdensity_fn)
        q, logp = state
        eng = get_engine(q, logdensity_fn)
        if not isinstance(logp, torch.Tensor):  # a stored log-density given as one number, as the reference allows
            logp = torch.full((eng.C,), float(logp), dtype=torch.float32, device=eng.device)
        eng.ensure_rw_proposal(kind, self._dev(sigma, eng.device), self._dev(mean, eng.device))
        pa = torch.empty(eng.C, dtype=torch.float32, device=eng.device)
        acc = torch.empty(eng.C, dtype=torch.uint8, device=eng.device)
        out = (q, logp) if self.inplace else None
        qo, lo = eng.rw_step(rng_key, q, logp, correct, out=out,
                             info_fields=dict(acceptance_rate=pa, is_accepted=acc), chain_offset=self.chain_offset)
        new = RWState(qo, lo)
        return new, RWInfo(pa, acc.bool(), new)


def build_additive_step(inplace: bool = False, chain_offset: int = 0):
    """random_walk.py build_additive_step: ``kernel(rng_key, state, logdensity_fn, random_step)`` with ``random_step``
    a :func:`normal` descriptor.  ``inplace=True`` overwrites the input state's tensors; ``chain_offset`` is the global
    index of this process's first chain when one shared ``rng_key`` is split across GPUs."""
    run = _Runner(inplace, chain_offset)

    def kernel(rng_key, state, logdensity_fn, random_step):
        return run(rng_key, state, logdensity_fn, random_step, "random_step")

    return kernel


def additive_step_random_walk(logdensity_fn, random_step):
    """random_walk.py additive_step_random_walk: ``blackjax.additive_step_random_walk``."""
    _proposal_of(random_step, "random_step")
    return build_sampling_algorithm(build_additive_step(), init, logdensity_fn, kernel_args=(random_step,))


def normal_random_walk(logdensity_fn, sigma):
    """random_walk.py normal_random_walk: ``blackjax.additive_step_random_walk.normal_random_walk``."""
    return additive_step_random_walk(logdensity_fn, normal(sigma))


def build_irmh(inplace: bool = False, chain_offset: int = 0):
    """random_walk.py build_irmh: ``kernel(rng_key, state, logdensity_fn, proposal_distribution,
    proposal_logdensity_fn=None)`` with a :func:`gaussian_distribution` and, optionally, its
    :func:`gaussian_logdensity`.  ``inplace`` and ``chain_offset`` as in :func:`build_additive_step`."""
    run = _Runner(inplace, chain_offset)

    def kernel(rng_key, state, logdensity_fn, proposal_distribution, proposal_logdensity_fn=None):
        return run(rng_key, state, logdensity_fn, proposal_distribution, "proposal_distribution",
                   proposal_logdensity_fn)

    return kernel


def irmh_as_top_level_api(logdensity_fn, proposal_distribution, proposal_logdensity_fn=None):
    """random_walk.py irmh_as_top_level_api: ``blackjax.irmh``."""
    _correct_of(_proposal_of(proposal_distribution, "proposal_distribution"), proposal_logdensity_fn)
    return build_sampling_algorithm(build_irmh(), init, logdensity_fn,
                                    kernel_args=(proposal_distribution, proposal_logdensity_fn))


def build_rmh(inplace: bool = False, chain_offset: int = 0):
    """random_walk.py build_rmh: ``kernel(rng_key, state, logdensity_fn, transition_generator,
    proposal_logdensity_fn=None)`` with a :func:`gaussian_proposal` and, for a position-independent one, optionally
    its :func:`gaussian_logdensity`.  ``inplace`` and ``chain_offset`` as in :func:`build_additive_step`."""
    run = _Runner(inplace, chain_offset)

    def kernel(rng_key, state, logdensity_fn, transition_generator, proposal_logdensity_fn=None):
        return run(rng_key, state, logdensity_fn, transition_generator, "transition_generator", proposal_logdensity_fn)

    return kernel


def rmh_as_top_level_api(logdensity_fn, proposal_generator, proposal_logdensity_fn=None):
    """random_walk.py rmh_as_top_level_api: ``blackjax.rmh``."""
    _correct_of(_proposal_of(proposal_generator, "transition_generator"), proposal_logdensity_fn)
    return build_sampling_algorithm(build_rmh(), init, logdensity_fn,
                                    kernel_args=(proposal_generator, proposal_logdensity_fn))
