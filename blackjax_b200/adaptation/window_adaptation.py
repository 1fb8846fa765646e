"""Stan-style window adaptation (step-size dual averaging + diagonal Welford mass matrix) for the
batched HMC/NUTS kernels.

Mirrors ``blackjax.window_adaptation`` (blackjax/adaptation/window_adaptation.py:296-444 ->
staged_adaptation.py:111-307,731-754,864-874,906-966).  Two modes:

* ``shared=False`` (default): every chain adapts its own (step_size, inverse mass matrix) -- what a
  BlackJAX user gets from ``jax.vmap(warmup.run)``.  Device-resident per-chain dual averaging and
  Welford accumulators (libbjx ``bjx_da_*`` / ``bjx_welford_*``); no communication.
* ``shared=True``: ONE step size and inverse mass matrix for all chains on all GPUs -- the
  reference's multi-chain path (staged_adaptation.py:906-966): dual averaging is fed
  ``mean(acceptance_rate)`` (one update per warm-up step, :153-171) and the mass matrix comes from the
  chain-pooled Chan-Golub-LeVeque merge (metric_buffers.py:334-420).  Each GPU reduces its chains to a
  ``(sum accept, n, mean[D], M2[D])`` block (``bjx_pooled_stats``); the blocks are exchanged with ONE
  all-gather per warm-up step and merged identically on every rank.
"""
import math
from typing import NamedTuple

import torch

from .. import random as bjx_random
from .._lib import check, lib, ptr
from ..base import AdaptationAlgorithm, AdaptationResults


def slow_windows(num_steps, initial_buffer_size=75, final_buffer_size=50, first_window_size=25):
    """Half-open [start, end) ranges of the slow (mass-matrix) windows of Stan's warm-up: windows double in size until
    the next doubled window would not fit before the final fast buffer, and the last one absorbs the remainder
    (same arithmetic as blackjax/adaptation/staged_adaptation.py:357-395)."""
    if num_steps < 20:
        return []
    if initial_buffer_size + first_window_size + final_buffer_size > num_steps:
        initial_buffer_size = int(0.15 * num_steps)
        final_buffer_size = int(0.1 * num_steps)
        first_window_size = num_steps - initial_buffer_size - final_buffer_size
    stop = num_steps - final_buffer_size
    windows, start, size = [], initial_buffer_size, first_window_size
    while start < stop:
        room = stop - start
        end = start + size if 3 * size <= room else stop
        windows.append((start, end))
        start, size = end, 2 * size
    return windows


def build_schedule(num_steps, initial_buffer_size=75, final_buffer_size=50, first_window_size=25):
    """Per-step (stage, is_middle_window_end) pairs, stage 0 = fast (step size only), 1 = slow (step size + mass
    matrix); the last step of every slow window carries True (blackjax/adaptation/staged_adaptation.py:315-405)."""
    schedule = [(0, False)] * num_steps
    for start, end in slow_windows(num_steps, initial_buffer_size, final_buffer_size, first_window_size):
        for t in range(start, end):
            schedule[t] = (1, t == end - 1)
    return schedule


# ---- host-side float32 dual averaging for the shared-epsilon mode (one scalar state) -----------------
class _DA(NamedTuple):
    log_step: float
    log_step_avg: float
    step: int
    avg_error: float
    mu: float


def _f32(x):
    return torch.tensor(x, dtype=torch.float32).item()


def _da_init(eps):
    return _DA(_f32(math.log(_f32(eps))), 0.0, 1, 0.0, _f32(math.log(_f32(10.0 * _f32(eps)))))


def _da_update(s, acceptance_rate, target, t0=10, gamma=0.05, kappa=0.75):
    """optimizers/dual_averaging.py:101-123 in float32 (torch CPU scalars; O(1) host work)."""
    f = lambda v: torch.tensor(v, dtype=torch.float32)
    log_step, avg, step, avg_error, mu = (f(s.log_step), f(s.log_step_avg), s.step, f(s.avg_error), f(s.mu))
    gradient = f(target) - f(acceptance_rate)
    reg_step = f(float(step + t0))
    eta_t = torch.pow(f(float(step)), f(-kappa))
    avg_error = (f(1.0) - (f(1.0) / reg_step)) * avg_error + gradient / reg_step
    log_x = mu - (torch.sqrt(f(float(step))) / f(gamma)) * avg_error
    log_x_avg = eta_t * log_step + (f(1.0) - eta_t) * avg
    return _DA(log_x.item(), log_x_avg.item(), step + 1, avg_error.item(), s.mu)


def _cross(delta, dense):
    return torch.outer(delta, delta) if dense else delta * delta


def cgl_merge_blocks(blocks, dim=None):
    """Chan-Golub-LeVeque merge of per-GPU blocks [G, 2+2D] (diagonal M2) or [G, 2+D+D*D] (dense M2, pass ``dim``)
    -> (sum_accept, n, mean[D], M2)  (metric_buffers.py:334-393), sequential in rank order so every rank computes
    identical bits."""
    dense = dim is not None and blocks.shape[1] == 2 + dim + dim * dim and dim > 1
    D = dim if dim is not None else (blocks.shape[1] - 2) // 2
    shape = (D, D) if dense else (D,)
    acc = blocks[0, 0].clone()
    n = blocks[0, 1].clone()
    mean = blocks[0, 2:2 + D].clone()
    m2 = blocks[0, 2 + D:].reshape(shape).clone()
    for gidx in range(1, blocks.shape[0]):
        nb = blocks[gidx, 1]
        mb = blocks[gidx, 2:2 + D]
        m2b = blocks[gidx, 2 + D:].reshape(shape)
        n_ab = n + nb
        delta = mb - mean
        mean = mean + delta * (nb / n_ab)
        m2 = m2 + m2b + _cross(delta, dense) * (n * nb / n_ab)
        n = n_ab
        acc = acc + blocks[gidx, 0]
    return acc, n, mean, m2


def _allgather_stats(block, group):
    """ONE all-gather of the per-GPU summary block (NCCL over NVLink on GPUs, gloo in the CPU tests)."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return block[None]
    world = dist.get_world_size(group)
    flat = block.contiguous().view(-1)
    out = torch.empty(world * flat.numel(), dtype=block.dtype, device=block.device)
    dist.all_gather_into_tensor(out, flat, group=group)
    return out.view((world,) + tuple(block.shape))


def native_run_inputs(eng, state, rng_key, chain_offset, is_nuts, extra_parameters, leapfrog_counter):
    """What the native warm-up loops (bjx_adapt_shared_run, bjx_lowrank_window_run) take besides their recipe's state:
    ``(max_num_doublings, num_integration_steps, q, logp, grad, acceptance_scratch, steps_scratch, rng_key)`` -- the
    transition's length argument with the other one 0, clones of ``state`` that the loop advances in place, the
    per-chain scratch arrays (the leapfrog counts only when they are accumulated) and the contiguous device key, which
    the engine is told is one step key shared by the chains from global index ``chain_offset``."""
    mnd = int(extra_parameters.get("max_num_doublings", 10)) if is_nuts else 0
    nis = 0 if is_nuts else int(extra_parameters["num_integration_steps"])
    q, lp, g = state.position.clone(), state.logdensity.clone(), state.logdensity_grad.clone()
    acc_scratch = torch.empty(eng.C, dtype=torch.float32, device=eng.device)
    steps_scratch = torch.empty(eng.C, dtype=torch.int32, device=eng.device) if leapfrog_counter is not None else None
    rk = rng_key.to(eng.device).contiguous()
    eng._key_mode(rk, chain_offset)
    return mnd, nis, q, lp, g, acc_scratch, steps_scratch, rk


def window_adaptation(algorithm, logdensity_fn, is_mass_matrix_diagonal: bool = True,
                      initial_step_size: float = 1.0, target_acceptance_rate: float = 0.80, shared: bool = False,
                      process_group=None, **extra_parameters):
    """blackjax/adaptation/window_adaptation.py:296-444.  ``algorithm`` is ``blackjax_b200.hmc`` or
    ``blackjax_b200.nuts``; ``extra_parameters`` go to the kernel (``num_integration_steps`` /
    ``max_num_doublings``).  Returns an :class:`AdaptationAlgorithm` with ``run(rng_key, position, num_steps)``."""
    dense = not is_mass_matrix_diagonal
    def run(rng_key, position, num_steps: int = 1000, _leapfrog_counter=None):
        from .._engine import get_engine
        position = position.contiguous()
        C, D = position.shape
        dev = position.device
        state = algorithm.init(position, logdensity_fn)
        # the engine the transition kernel resolves to (nuts.build_kernel: depth max(10, max_num_doublings))
        eng = get_engine(position, logdensity_fn, max_tree_depth=max(10, extra_parameters.get("max_num_doublings", 10)))
        schedule = build_schedule(num_steps)
        history = []
        import torch.distributed as dist
        world, rank = 1, 0
        if shared and dist.is_available() and dist.is_initialized():
            world, rank = dist.get_world_size(process_group), dist.get_rank(process_group)
        if shared and not dense and position.is_cuda:
            # ---- device-resident shared adaptation (libbjx bjx_adapt_shared_*): block statistics, ONE NCCL all-gather,
            # merge + dual averaging + window bookkeeping on the device; no host round trip per warm-up step --------
            from .._comm import nccl_comm
            comm, n_ranks, rank = nccl_comm(dev, process_group)
            L = lib()
            st = torch.empty(L.bjx_adapt_shared_state_floats(C, D, n_ranks), dtype=torch.float32, device=dev)
            eps_c = torch.empty(C, dtype=torch.float32, device=dev)
            imm = torch.empty(D, dtype=torch.float32, device=dev)
            eps_hist = torch.empty(num_steps, dtype=torch.float32, device=dev)
            check(L.bjx_adapt_shared_init(eng.h, ptr(st), float(initial_step_size), ptr(eps_c), ptr(imm)), eng.h)
            eng._imm, eng._imm_key = imm, (imm.data_ptr(), tuple(imm.shape), imm._version, str(imm.device))
            # the loop itself runs in libbjx (bjx_adapt_shared_run): transition, block statistics, all-gather, device-side
            # update per warm-up step, nothing waits for the device.  Chain c of this rank uses
            # split(step_key, C_global)[rank * C + c] (staged_adaptation.py:920), derived inside the transition kernel
            sched = bytes(int(stage) | (int(window_end) << 1) for stage, window_end in schedule)
            mnd, nis, q, lp, g, acc_scratch, steps_scratch, rk = native_run_inputs(
                eng, state, rng_key, rank * C, "num_integration_steps" not in extra_parameters, extra_parameters,
                _leapfrog_counter)
            check(L.bjx_adapt_shared_run(eng.h, comm, n_ranks, ptr(rk), sched, int(num_steps), ptr(q), ptr(lp), ptr(g), ptr(st),
                                         ptr(eps_c), ptr(imm), float(target_acceptance_rate), mnd, nis, ptr(eps_hist),
                                         ptr(acc_scratch), ptr(steps_scratch), ptr(_leapfrog_counter)), eng.h)
            imm.add_(0.0)  # version bump: the kernels' metric cache follows the contents the device rewrote
            state = type(state)(q, lp, g)
            step = torch.empty(1, dtype=torch.float32, device=dev)
            check(L.bjx_adapt_shared_final(eng.h, ptr(st), ptr(step)), eng.h)
            step_size = float(step.item())   # the one host read of the warm-up
            parameters = {"step_size": step_size, "inverse_mass_matrix": imm, **extra_parameters}
            return AdaptationResults(state, parameters), eps_hist.cpu()
        # shared mode: one step key per warm-up step; chain c of this rank uses split(step_key, C_global)[rank*C + c]
        # (staged_adaptation.py:920), derived inside the transition kernel
        mcmc_kernel = algorithm.build_kernel(chain_offset=rank * C)
        if shared:
            step_keys = bjx_random.split(rng_key.to(dev), num_steps)
            da = _da_init(initial_step_size)
            eps = _f32(initial_step_size)
            m2_shape = (D, D) if dense else (D,)
            imm = torch.eye(D, dtype=torch.float32, device=dev) if dense else torch.ones(D, dtype=torch.float32, device=dev)
            w_n, w_mean, w_m2 = 0.0, torch.zeros(D, device=dev), torch.zeros(m2_shape, device=dev)
            stats = torch.empty(2 + D + (D * D if dense else D), dtype=torch.float32, device=dev)
            pooled = lib().bjx_pooled_stats_dense if dense else lib().bjx_pooled_stats
            for t, (stage, window_end) in enumerate(schedule):
                state, info = mcmc_kernel(step_keys[t], state, logdensity_fn, eps, imm, **extra_parameters)
                check(pooled(eng.h, ptr(state.position), ptr(info.acceptance_rate), ptr(stats)), eng.h)
                blocks = _allgather_stats(stats, process_group)
                acc_sum, n_b, mean_b, m2_b = cgl_merge_blocks(blocks, D)
                if stage == 1:  # CGL-merge this step's pooled block into the window accumulator
                    if w_n == 0.0:
                        w_n, w_mean, w_m2 = float(n_b), mean_b, m2_b
                    else:
                        nb = float(n_b)
                        n_ab = w_n + nb
                        delta = mean_b - w_mean
                        w_mean = w_mean + delta * (nb / n_ab)
                        w_m2 = w_m2 + m2_b + _cross(delta, dense) * (w_n * nb / n_ab)
                        w_n = n_ab
                da = _da_update(da, (acc_sum / n_b).item(), target_acceptance_rate)
                eps = _f32(math.exp(da.log_step))
                if window_end:  # mass_matrix.py:335-357 + staged_adaptation.py:233-249
                    cov = w_m2 / (w_n - 1.0)
                    reg = (5.0 / (w_n + 5.0)) * 1e-3
                    imm = (w_n / (w_n + 5.0)) * cov + (reg * torch.eye(D, device=dev) if dense else reg)
                    imm = imm.to(torch.float32).contiguous()
                    w_n, w_mean, w_m2 = 0.0, torch.zeros(D, device=dev), torch.zeros(m2_shape, device=dev)
                    da = _da_init(_f32(math.exp(da.log_step_avg)))
                    eps = _f32(math.exp(da.log_step))
                history.append(eps)
            step_size = _f32(math.exp(da.log_step_avg))
            parameters = {"step_size": step_size, "inverse_mass_matrix": imm, **extra_parameters}
            return AdaptationResults(state, parameters), history
        # ---- per-chain adaptation, all state on the device ------------------------------------------------
        if rng_key.ndim == 1:
            chain_keys = bjx_random.split(rng_key.to(dev), C)
        else:
            chain_keys = rng_key
        keys = bjx_random.split(chain_keys, num_steps)                      # [C, T, 2]   (util.py:203 per chain)
        keys = keys.transpose(0, 1).contiguous()                            # [T, C, 2]
        da_state = torch.empty(C, 5, dtype=torch.float32, device=dev)
        eps = torch.full((C,), float(initial_step_size), dtype=torch.float32, device=dev)
        check(lib().bjx_da_init(eng.h, ptr(da_state), ptr(eps), ptr(eps)), eng.h)
        if dense:  # one dense matrix per chain (what jax.vmap(warmup.run) carries with is_mass_matrix_diagonal=False)
            if D > 64:
                raise NotImplementedError("per-chain dense adaptation is built for dim <= 64 ([C, D, D] metrics); use "
                                          "shared=True (pooled dense metric, any dim) beyond")
            imm = torch.eye(D, dtype=torch.float32, device=dev).repeat(C, 1, 1).contiguous()
            w_m2 = torch.zeros(C, D, D, dtype=torch.float32, device=dev)
            wf_update, wf_final = lib().bjx_welford_dense_update, lib().bjx_welford_dense_final
        else:
            imm = torch.ones(C, D, dtype=torch.float32, device=dev)
            w_m2 = torch.zeros(C, D, dtype=torch.float32, device=dev)
            wf_update, wf_final = lib().bjx_welford_update, lib().bjx_welford_final
        w_mean = torch.zeros(C, D, dtype=torch.float32, device=dev)
        w_n = 0
        for t, (stage, window_end) in enumerate(schedule):
            state, info = mcmc_kernel(keys[t], state, logdensity_fn, eps, imm, **extra_parameters)
            if stage == 1:
                w_n += 1
                check(wf_update(eng.h, ptr(state.position), ptr(w_mean), ptr(w_m2), w_n), eng.h)
            check(lib().bjx_da_update(eng.h, ptr(da_state), ptr(info.acceptance_rate), float(target_acceptance_rate),
                                      ptr(eps)), eng.h)
            if window_end:
                new_imm = torch.empty_like(imm)
                check(wf_final(eng.h, ptr(w_mean), ptr(w_m2), w_n, ptr(new_imm)), eng.h)
                imm = new_imm   # new tensor identity => the kernel re-derives mass_matrix_sqrt
                w_n = 0
                check(lib().bjx_da_reset(eng.h, ptr(da_state), ptr(eps)), eng.h)
        step_size = torch.empty(C, dtype=torch.float32, device=dev)
        check(lib().bjx_da_final(eng.h, ptr(da_state), ptr(step_size)), eng.h)
        parameters = {"step_size": step_size, "inverse_mass_matrix": imm, **extra_parameters}
        return AdaptationResults(state, parameters), history

    return AdaptationAlgorithm(run)
