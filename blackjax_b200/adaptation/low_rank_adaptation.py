"""Low-rank window adaptation for HMC / NUTS: Stan's window schedule with the Fisher-divergence low-rank metric.

Mirrors ``blackjax.window_adaptation_low_rank`` (blackjax/adaptation/low_rank_adaptation.py:458-652) with
``buffer_policy="reset"``, pooled over chains: ONE step size and ONE low-rank inverse mass matrix
``M^-1 = diag(sigma) (I + U (diag(lam) - I) U^T) diag(sigma)`` for all chains -- the observation model of the
reference's multi-chain path (staged_adaptation.py:906-966).  Dual averaging is fed the mean acceptance rate of all
chains, and at every window end the estimator (_compute_low_rank_metric, metric_estimators.py:618-808) sees the
stacked draws and gradients of all chains.  With one chain this is the reference's single-chain warm-up.

The whole loop runs in libbjx (``bjx_lowrank_window_run``): per step one transition, the windowed covariance folds of
the draws and the gradients, the dual-averaging update and, at a window end, the estimator and the in-place install of
the new metric -- all on the device, with no host round trip.  Built for dim <= 512 and max_rank <= 16 on one GPU.
"""
from typing import NamedTuple

import torch

from .._lib import check, lib, ptr
from ..base import AdaptationAlgorithm, AdaptationResults
from ..mcmc.metrics import LowRankMetric
from .window_adaptation import build_schedule, native_run_inputs

__all__ = ["LowRankWindowInfo", "build_growing_window_schedule", "window_adaptation_low_rank"]

MAX_DIM, MAX_RANK = 512, 16


def build_growing_window_schedule(num_steps, early_window=0.3, step_size_window=0.15, early_window_size=10,
                                  window_size=80, window_growth=1.5):
    """Per-step (stage, window_end) pairs of nutpie's proportional, geometrically growing schedule
    (low_rank_adaptation.py:310-450): fixed windows of ``early_window_size`` over the first ``early_window`` of the
    steps, then windows growing by ``window_growth`` from ``window_size``; a window whose successor would not fit before
    the final step-size-only phase (the last ``step_size_window`` of the steps) absorbs the rest (``is_late``)."""
    if num_steps < 20:
        return [(0, False)] * num_steps
    final_buffer_size = max(int(round(step_size_window * num_steps)), 1)
    final_buffer_start = num_steps - final_buffer_size
    early_end = min(max(int(round(early_window * num_steps)), 1), final_buffer_start)
    schedule = []
    pos = 0
    while pos < early_end:
        size = min(early_window_size, early_end - pos)
        schedule += [(1, False)] * (size - 1) + [(1, True)]
        pos += size
    current = window_size
    while pos < final_buffer_start:
        nxt = max(current + 1, int(round(current * window_growth)))
        size = final_buffer_start - pos if (pos + current) + nxt > final_buffer_start else current
        schedule += [(1, False)] * (size - 1) + [(1, True)]
        pos += size
        if size != current:
            break
        current = nxt
    schedule += [(0, False)] * (num_steps - pos)
    return schedule


def buffer_size(num_steps):
    """Rows of the reference's circular draw buffer under buffer_policy="reset" (low_rank_adaptation.py:604-605)."""
    return min(2 * max(num_steps // 5, 128), max(num_steps, 1))


def schedule_bytes(schedule, num_steps):
    """stage | window_end << 1 | retained << 2 per step.  A slow step is retained when the reference's buffer of
    ``buffer_size(num_steps)`` rows still holds it at its window's end: the last min(len, B) steps of a window."""
    pairs = [(int(s), bool(e)) for s, e in (tuple(p) for p in schedule)]
    if len(pairs) != num_steps:
        raise ValueError(f"schedule_fn returned {len(pairs)} steps, expected {num_steps}")
    B = buffer_size(num_steps)
    out = [0] * num_steps
    start = None
    for t, (stage, end) in enumerate(pairs):
        if stage not in (0, 1):
            raise ValueError(f"schedule stage must be 0 or 1, got {stage} at step {t}")
        if end and stage != 1:
            raise ValueError(f"a window ends on a slow-stage step; step {t} is fast")
        if stage == 1 and start is None:
            start = t
        if stage == 0 and start is not None:     # slow steps that no window end closes: never read
            start = None
        out[t] = stage | (int(end) << 1)
        if end:
            for u in range(max(start, t + 1 - B), t + 1):
                out[u] |= 4
            start = None
    return bytes(out)


class LowRankWindowInfo(NamedTuple):
    """What ``run`` returns next to the results: the last warm-up state, mu* of the last window end, the per-step step
    sizes (device tensor) and the eigensolver's diagnostics over both top-k solves of every window end."""

    state: object
    mu_star: torch.Tensor
    step_size: torch.Tensor
    eigensolver_iterations: int        # largest over the solves of the last window end
    eigensolver_residual: float        # largest relative residual ||S u - lam u|| / max lam of those solves
    eigensolver_not_converged: bool    # sticky: any solve stopped at its iteration cap


class _LowRankWindow:
    """Device state of bjx_lowrank_window_* for an engine of C chains and D dims, rank k.  ``install`` puts the initial
    metric (ones, zeros, ones) into the handle; every window end rewrites it in place."""

    def __init__(self, eng, k):
        self.eng, self.k = eng, k
        n = lib().bjx_lowrank_window_state_floats(eng.C, eng.D, k)
        if n == 0:
            raise ValueError(f"window_adaptation_low_rank is built for dim <= {MAX_DIM} and 1 <= max_rank <= {MAX_RANK}")
        self.state = torch.empty(n, dtype=torch.float32, device=eng.device)
        self.eps_c = torch.empty(eng.C, dtype=torch.float32, device=eng.device)

    def install(self, initial_step_size):
        D, k, dev = self.eng.D, self.k, self.eng.device
        self._init_metric = LowRankMetric(torch.ones(D, device=dev), torch.zeros(D, k, device=dev), torch.ones(k, device=dev))
        self.eng.ensure_metric(self._init_metric)    # BjxError when the transitions do not run on the warp kernels
        check(lib().bjx_lowrank_window_init(self.eng.h, ptr(self.state), float(initial_step_size), ptr(self.eps_c)),
              self.eng.h)
        self.eng._imm_key = None   # the device rewrites the installed block: no tensor's content matches it any more

    def update(self, q, g, acceptance_rate, sched_byte, target, gamma, cutoff, eps_hist=None):
        check(lib().bjx_lowrank_window_update(self.eng.h, ptr(self.state), ptr(q), ptr(g), ptr(acceptance_rate),
                                              int(sched_byte), float(target), float(gamma), float(cutoff),
                                              ptr(self.eps_c), ptr(eps_hist)), self.eng.h)

    def final(self):
        """(step size [1], mu* [D], LowRankMetric) as new device tensors."""
        D, k, dev = self.eng.D, self.k, self.eng.device
        step, mu, sigma, lam = (torch.empty(n, dtype=torch.float32, device=dev) for n in (1, D, D, k))
        U = torch.empty(D, k, dtype=torch.float32, device=dev)
        check(lib().bjx_lowrank_window_final(self.eng.h, ptr(self.state), ptr(step), ptr(mu), ptr(sigma), ptr(U),
                                             ptr(lam)), self.eng.h)
        return step, mu, LowRankMetric(sigma, U, lam)

    def diagnostics(self):
        h = self.state[32:64].view(2, 16).cpu().tolist()
        return (int(max(r[1] for r in h)), float(max(r[2] for r in h)), bool(any(r[3] for r in h)))


def _check_process_group(process_group):
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(process_group) > 1:
        raise NotImplementedError("window_adaptation_low_rank runs on one GPU; a process group of more than one rank "
                                  "is not supported")


def window_adaptation_low_rank(algorithm, logdensity_fn, max_rank: int = 10, initial_step_size: float = 1.0,
                               target_acceptance_rate: float = 0.80, gamma: float = 1e-5, cutoff: float = 2.0,
                               schedule_fn=build_schedule, buffer_policy: str = "reset", gradient_based_init: bool = False,
                               process_group=None, **extra_parameters):
    """blackjax/adaptation/low_rank_adaptation.py:458-652, pooled over chains.  ``algorithm`` is ``blackjax_b200.nuts``
    (``max_num_doublings``) or ``blackjax_b200.hmc`` (``num_integration_steps``).  ``run(rng_key, position[C, D],
    num_steps=1000)`` returns ``(AdaptationResults(state, parameters), LowRankWindowInfo)`` with
    ``parameters = {"step_size": float, "inverse_mass_matrix": LowRankMetric(sigma, U, lam), **extra_parameters}`` and
    every chain's state re-initialised at mu* = x_bar + sigma^2 g_bar of the last window end (zeros if none ended)."""
    import blackjax_b200 as bj
    if buffer_policy == "accumulating":
        raise NotImplementedError("buffer_policy='accumulating' is not built; use 'reset'")
    if buffer_policy != "reset":
        raise ValueError(f"buffer_policy must be 'reset' or 'accumulating', got {buffer_policy!r}")
    if gradient_based_init:
        raise NotImplementedError("gradient_based_init=True is not built for the pooled warm-up")
    if not 1 <= int(max_rank) <= MAX_RANK:
        raise ValueError(f"max_rank must be in [1, {MAX_RANK}], got {max_rank}")
    if not (gamma > 0 and cutoff > 0):
        raise ValueError("gamma and cutoff must be positive")
    if "integrator" in extra_parameters:
        raise ValueError("window_adaptation_low_rank runs the kernels' velocity Verlet integrator; other integrators "
                         "are not supported")
    if algorithm is bj.nuts:
        is_nuts = True
    elif algorithm is bj.hmc:
        is_nuts = False
        if "num_integration_steps" not in extra_parameters:
            raise ValueError("hmc needs num_integration_steps")
    else:
        raise ValueError("window_adaptation_low_rank supports blackjax_b200.nuts and blackjax_b200.hmc")
    k = int(max_rank)

    def run(rng_key, position, num_steps: int = 1000, _leapfrog_counter=None):
        from .._engine import get_engine
        _check_process_group(process_group)
        position = position.contiguous()
        if position.ndim != 2 or not position.is_cuda:
            raise ValueError("position must be a [num_chains, dim] CUDA tensor")
        C, D = position.shape
        if D > MAX_DIM:
            raise ValueError(f"window_adaptation_low_rank is built for dim <= {MAX_DIM}, got {D}")
        dev = position.device
        sched = schedule_bytes(schedule_fn(num_steps), num_steps)
        state = algorithm.init(position, logdensity_fn)
        eng = get_engine(position, logdensity_fn, max_tree_depth=max(10, int(extra_parameters.get("max_num_doublings", 10))))
        lw = _LowRankWindow(eng, k)
        lw.install(initial_step_size)
        eps_hist = torch.empty(num_steps, dtype=torch.float32, device=dev)
        mnd, nis, q, lp, g, acc_scratch, steps_scratch, rk = native_run_inputs(eng, state, rng_key, 0, is_nuts,
                                                                                extra_parameters, _leapfrog_counter)
        check(lib().bjx_lowrank_window_run(eng.h, ptr(rk), sched, int(num_steps), ptr(q), ptr(lp), ptr(g), ptr(lw.state),
                                           ptr(lw.eps_c), float(target_acceptance_rate), float(gamma), float(cutoff), mnd,
                                           nis, ptr(eps_hist), ptr(acc_scratch), ptr(steps_scratch),
                                           ptr(_leapfrog_counter)), eng.h)
        last = type(state)(q, lp, g)
        step, mu_star, metric = lw.final()
        for t in metric:
            t.add_(0.0)    # version bump: the kernels' metric cache follows contents the device wrote
        step_size = float(step.item())
        iters, resid, noconv = lw.diagnostics()
        new_state = algorithm.init(mu_star[None].expand(C, D).contiguous(), logdensity_fn)   # :643-650
        parameters = {"step_size": step_size, "inverse_mass_matrix": metric, **extra_parameters}
        info = LowRankWindowInfo(last, mu_star, eps_hist, iters, resid, noconv)
        return AdaptationResults(new_state, parameters), info

    return AdaptationAlgorithm(run)
