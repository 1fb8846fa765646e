"""MEADS warm-up for generalized HMC: cross-chain adaptation of step size, momentum scale, persistence and slice drift.

Mirrors ``blackjax.meads_adaptation`` (blackjax/adaptation/meads_adaptation.py:316-784) for its default configuration
(``low_rank_rank=None``: one diagonal momentum scale per fold).  Per warm-up step: ``bjx_meads_update`` (fold statistics,
``maximum_eigenvalue`` of the preconditioned gradients / positions, parameters rolled to the next fold -- four launches,
nothing read back), one ``bjx_ghmc_step`` of every chain with its fold's parameters (fold ``t mod K`` frozen), and every
K steps ``bjx_permutation`` + ``bjx_gather_rows`` (``jax.random.permutation`` of all chains).  The loop never
synchronises with the host.

With ``low_rank_rank=k`` (MEADS-LRD, :459-784) every chain samples with ONE low-rank metric per step instead of the fold
scales: ``bjx_meads_lrd_update`` replaces ``bjx_meads_update`` (it also folds the positions into the windowed covariance
accumulator, runs the on-device eigensolver and rewrites the handle's low-rank metric in place), and the run returns a
``LowRankMetric`` as ``momentum_inverse_scale``.  Built for dim <= 512 and k <= 16 on one GPU.
"""
import warnings
from typing import NamedTuple

import torch

from .. import random as bjx_random
from .._lib import BjxError, check, lib, ptr
from ..base import AdaptationAlgorithm, AdaptationResults
from ..mcmc import ghmc
from ..mcmc.metrics import LowRankMetric

__all__ = ["MEADSAdaptationState", "base", "maximum_eigenvalue", "meads_adaptation"]


class MEADSAdaptationState(NamedTuple):
    """meads_adaptation.py:31-53: per-fold parameters (device tensors)."""

    current_iteration: int
    step_size: torch.Tensor        # [K]
    position_sigma: torch.Tensor   # [K, D]
    alpha: torch.Tensor            # [K]
    delta: torch.Tensor            # [K]


class _Folds:
    """Device buffers of bjx_meads_update for (C chains, D dims, K folds)."""

    def __init__(self, eng, K):
        L = lib()
        self.eng, self.K = eng, K
        dev = eng.device
        self.state = torch.empty(L.bjx_meads_state_floats(K, eng.D), dtype=torch.float32, device=dev)
        self.scratch = torch.empty(L.bjx_meads_scratch_floats(eng.C, eng.D, K), dtype=torch.float32, device=dev)
        KD = K * eng.D
        self.step_size, self.alpha, self.delta = self.state[0:K], self.state[K:2 * K], self.state[2 * K:3 * K]
        self.sigma = self.state[3 * K:3 * K + KD].view(K, eng.D)
        self.imm = self.state[3 * K + KD:3 * K + 2 * KD].view(K, eng.D)
        self.msqrt = self.state[3 * K + 2 * KD:3 * K + 3 * KD].view(K, eng.D)

    def update(self, q, g, t, multiplier, slowdown):
        check(lib().bjx_meads_update(self.eng.h, ptr(q), ptr(g), self.K, int(t), float(multiplier), float(slowdown),
                                     ptr(self.state), ptr(self.scratch)), self.eng.h)

    def snapshot(self, t):
        return MEADSAdaptationState(t, self.step_size.clone(), self.sigma.clone(), self.alpha.clone(), self.delta.clone())


class _LowRank:
    """Device buffers of bjx_meads_lrd_update / bjx_meads_lrd_metric for (C chains, D dims, rank k, K folds).  The
    handle must hold a rank-k low-rank metric; ``install`` puts the fallback one there."""

    MAX_DIM, MAX_RANK = 512, 16
    ENGAGED, ITERS, RESID, NOCONV, ITERS_SUM, ITERS_MAX, SOLVES = range(7)   # header slots (include/bjx.h)

    def __init__(self, eng, k, K):
        L = lib()
        self.eng, self.k, self.K = eng, k, K
        dev, C, D = eng.device, eng.C, eng.D
        self.state = torch.zeros(L.bjx_meads_lrd_state_floats(C, D, k), dtype=torch.float32, device=dev)
        self.scratch = torch.empty(L.bjx_meads_lrd_scratch_floats(C, D, K), dtype=torch.float32, device=dev)
        self.header = self.state[:16]
        o = 16
        self.sigma = self.state[o:o + D]
        self.U = self.state[o + D:o + D + D * k].view(D, k)
        self.lam = self.state[o + D + D * k:o + D + D * k + k]

    def install(self):
        """The fallback metric (ones, eye(D, k), ones); each update rewrites it in place."""
        D, k, dev = self.eng.D, self.k, self.eng.device
        metric = LowRankMetric(torch.ones(D, device=dev), torch.eye(D, k, device=dev), torch.ones(k, device=dev))
        try:
            self.eng.ensure_metric(metric)
        except BjxError as e:
            raise NotImplementedError(f"meads_adaptation(low_rank_rank=...) needs a target whose transitions run on the "
                                      f"warp kernels with a low-rank metric: {e}") from None

    def update(self, folds, q, g, t, in_window, multiplier, slowdown):
        check(lib().bjx_meads_lrd_update(self.eng.h, ptr(q), ptr(g), self.K, int(t), int(bool(in_window)), float(multiplier),
                                         float(slowdown), ptr(folds.state), ptr(self.state), ptr(self.scratch)), self.eng.h)

    def metric(self, final_q):
        """The final parameters (:746-771) as a LowRankMetric of new device tensors."""
        D, k, dev = self.eng.D, self.k, self.eng.device
        sigma, U, lam = (torch.empty(s, dtype=torch.float32, device=dev) for s in ((D,), (D, k), (k,)))
        check(lib().bjx_meads_lrd_metric(self.eng.h, ptr(self.state), ptr(final_q), ptr(sigma), ptr(U), ptr(lam)), self.eng.h)
        return LowRankMetric(sigma, U, lam)

    def warn_if_not_converged(self):
        """One host read of the eigensolver's diagnostics, after the run: warn when any solve stopped at its cap."""
        h = self.header.cpu().tolist()
        if h[self.NOCONV]:
            solves = max(h[self.SOLVES], 1.0)
            warnings.warn(f"MEADS-LRD: the eigensolver stopped at its iteration cap in at least one of {int(h[self.SOLVES])} "
                          f"solves (mean {h[self.ITERS_SUM] / solves:.1f}, max {int(h[self.ITERS_MAX])} iterations; last "
                          f"relative residual {h[self.RESID]:.2e}); the low-rank metric may be inaccurate", RuntimeWarning,
                          stacklevel=3)


def _low_rank_limits(logdensity_fn, k, D):
    """This port's limits of MEADS-LRD (NotImplementedError), after the rank is clamped to D."""
    if D > _LowRank.MAX_DIM or k > _LowRank.MAX_RANK:
        raise NotImplementedError(f"meads_adaptation(low_rank_rank=...) is built for dim <= {_LowRank.MAX_DIM} and a rank "
                                  f"<= {_LowRank.MAX_RANK}; got dim {D}, rank {k}")
    if not getattr(logdensity_fn, "build_options", {}).get("dense_metric", True):
        raise NotImplementedError("meads_adaptation(low_rank_rank=...) needs the low-rank metric kernels: build the "
                                  "UserTarget with dense_metric=True")


def _engine_for(positions, logdensity_fn):
    from .._engine import get_engine
    eng = get_engine(positions, logdensity_fn)
    eng.ensure_metric(torch.ones(eng.D, dtype=torch.float32, device=eng.device))   # rows are passed per launch
    return eng


def maximum_eigenvalue(matrix):
    """meads_adaptation.py:787-817 for an ``[n, d]`` CUDA matrix (the fold-statistics kernels of ``bjx_meads_update`` on
    one explicit matrix); returned as a 0-d device tensor."""
    x = matrix.contiguous().float()
    n, d = x.shape
    eng = _scratch_engine(x)
    L = lib()
    out = torch.empty((), dtype=torch.float32, device=x.device)
    scratch = torch.empty(L.bjx_maximum_eigenvalue_scratch_floats(n, d), dtype=torch.float32, device=x.device)
    check(L.bjx_maximum_eigenvalue(eng.h, ptr(x), n, d, ptr(out), ptr(scratch)), eng.h)
    return out


def base(num_folds: int = 4, step_size_multiplier: float = 0.5, damping_slowdown: float = 1.0):
    """meads_adaptation.py:56-214: ``(init, update)`` over per-fold device parameters."""
    if num_folds < 1:
        raise ValueError(f"num_folds must be >= 1, got {num_folds}.")

    def compute_parameters(positions, logdensity_grad, current_iteration, logdensity_fn=None):
        """:97-152 -- all given chains as ONE fold: (step_size, position_sigma, alpha, delta)."""
        eng = _scratch_engine(positions)
        f = _Folds(eng, 1)
        f.update(positions.contiguous(), logdensity_grad.contiguous(), current_iteration, step_size_multiplier,
                 damping_slowdown)
        return f.step_size[0].clone(), f.sigma[0].clone(), f.alpha[0].clone(), f.delta[0].clone()

    def init(positions, logdensity_grad):
        eps, sd, alpha, delta = compute_parameters(positions, logdensity_grad, 0)
        return MEADSAdaptationState(0, eps.repeat(num_folds), sd[None].repeat(num_folds, 1), alpha.repeat(num_folds),
                                    delta.repeat(num_folds))

    def update(adaptation_state, positions, logdensity_grad, source_fold: int):
        """:172-214: the source fold's statistics become the parameters of fold ``source_fold + 1``."""
        target = (int(source_fold) + 1) % num_folds
        t = adaptation_state.current_iteration
        eps, sd, alpha, delta = compute_parameters(positions, logdensity_grad, t)
        ss, sg, al, de = (x.clone() for x in adaptation_state[1:])
        ss[target], sg[target], al[target], de[target] = eps, sd, alpha, delta
        return MEADSAdaptationState(t + 1, ss, sg, al, de)

    return init, update


def _scratch_engine(x):
    """A handle for target-independent statistics kernels on x's device with x's shape."""
    from .. import targets
    from .._engine import get_engine
    return get_engine(x, targets.StdNormal(x.shape[1]))


def meads_adaptation(logdensity_fn, num_chains: int, num_folds: int = 4, step_size_multiplier: float = 0.5,
                     damping_slowdown: float = 1.0, adaptation_info_fn=None, low_rank_rank=None,
                     low_rank_window_fraction: float = 0.5):
    """meads_adaptation.py:316-784.  ``run(rng_key, positions, num_steps)`` returns ``(AdaptationResults(last GHMCState,
    parameters), info)``; ``info`` is the list of what ``adaptation_info_fn(state, info, adaptation_state)`` returned per
    step (None: nothing is stored).  ``low_rank_rank=k`` adapts one rank-min(k, num_chains - 1, dim) low-rank metric
    for all chains (MEADS-LRD), estimated from the covariance of all chains' positions over the last
    ``low_rank_window_fraction`` of the steps; ``parameters["momentum_inverse_scale"]`` is then a ``LowRankMetric``."""
    if num_folds < 1:
        raise ValueError(f"num_folds must be >= 1, got {num_folds}.")
    if num_chains % num_folds != 0:
        raise ValueError(f"num_chains ({num_chains}) must be divisible by num_folds ({num_folds}).")
    low_rank_k = None
    if low_rank_rank is not None:                                # :467-487
        low_rank_k = min(int(low_rank_rank), num_chains - 1)
        if low_rank_k < 1:
            raise ValueError(f"low_rank_rank={low_rank_rank} cannot be honored: the low-rank metric is estimated from "
                             f"the full population of num_chains={num_chains} chains, and that estimate needs "
                             "num_chains - 1 >= 1. Increase num_chains.")
        if not 0.0 <= low_rank_window_fraction <= 1.0:
            raise ValueError(f"low_rank_window_fraction must be in [0.0, 1.0], got {low_rank_window_fraction}.")
    n_per_fold = num_chains // num_folds
    kernel = ghmc.build_kernel(inplace=True)

    def run(rng_key, positions, num_steps: int = 1000):
        positions = positions.contiguous()
        C, D = positions.shape
        if C != num_chains:
            raise ValueError("initial `positions` leading dimension must be equal to the `num_chains`")
        dev = positions.device
        lowrank = None
        if low_rank_k is not None:
            _low_rank_limits(logdensity_fn, min(low_rank_k, D), D)
        eng = _engine_for(positions, logdensity_fn)
        if low_rank_k is not None:
            lowrank = _LowRank(eng, min(low_rank_k, D), num_folds)
            lowrank.install()
        L = lib()
        k2 = bjx_random.split(rng_key.to(dev), 2).view(torch.int32)
        key_init, key_adapt = k2[0].contiguous(), k2[1].contiguous()
        state = ghmc.init(positions.clone(), logdensity_fn, bjx_random.split(key_init, C))
        folds = _Folds(eng, num_folds)
        first = _Folds(eng, 1)                                   # adapt_init: all chains, replicated (:154-170)
        first.update(state.position, state.logdensity_grad, 0, step_size_multiplier, damping_slowdown)
        folds.step_size.copy_(first.step_size.expand(num_folds))
        folds.alpha.copy_(first.alpha.expand(num_folds))
        folds.delta.copy_(first.delta.expand(num_folds))
        folds.sigma.copy_(first.sigma.expand(num_folds, D))
        keys = bjx_random.split(key_adapt, num_steps)
        spare = tuple(torch.empty_like(x) for x in state)
        perm = torch.empty(C, dtype=torch.int32, device=dev)
        perm_scratch = torch.empty(L.bjx_permutation_scratch_bytes(C), dtype=torch.uint8, device=dev)
        window_start = int(low_rank_window_fraction * num_steps)    # :723
        infos = []
        for t in range(num_steps):
            skip = ((t % num_folds) * n_per_fold, (t % num_folds + 1) * n_per_fold) if num_folds > 1 else (0, 0)
            if lowrank is None:
                folds.update(state.position, state.logdensity_grad, t, step_size_multiplier, damping_slowdown)
                rows = (folds.step_size, folds.alpha, folds.delta, folds.imm, folds.msqrt, n_per_fold, skip)
            else:                                                # one shared metric, in the handle (:549-568,644-667)
                lowrank.update(folds, state.position, state.logdensity_grad, t, t >= window_start, step_size_multiplier,
                               damping_slowdown)
                rows = (folds.step_size, folds.alpha, folds.delta, None, None, n_per_fold, skip)
            state, info = kernel(keys[t], state, logdensity_fn, None, None, None, None, _rows=rows)
            if num_folds > 1 and (t + 1) % num_folds == 0:     # shuffle_key = split(rng_key, C + 1)[C]  (:503-504,675-683)
                check(L.bjx_permutation(eng.h, ptr(keys[t]), C, C, ptr(perm), ptr(perm_scratch)), eng.h)
                for src, dst in zip(state, spare):
                    width = src.shape[1] if src.ndim == 2 else 1
                    check(L.bjx_gather_rows(eng.h, ptr(perm), ptr(src), ptr(dst), C, width), eng.h)
                state, spare = ghmc.GHMCState(*spare), tuple(state)
            if adaptation_info_fn is not None:
                infos.append(adaptation_info_fn(state, info, folds.snapshot(t + 1)))
        last = folds.snapshot(num_steps)
        parameters = {
            "step_size": last.step_size.mean(),
            "momentum_inverse_scale": (last.position_sigma.mean(dim=0) if lowrank is None
                                       else lowrank.metric(state[0].contiguous())),
            "alpha": last.alpha.mean(),
            "delta": last.delta.mean(),
        }
        if lowrank is not None:
            lowrank.warn_if_not_converged()
        return AdaptationResults(ghmc.GHMCState(*state), parameters), infos

    return AdaptationAlgorithm(run)
