"""Float32 restatement of adjusted MCLMC's tuner (blackjax/adaptation/adjusted_mclmc_adaptation.py:26-507, with
dual_averaging_adaptation of step_size.py:65-150 and incremental_value_update of util.py:291-319), batched over independent
chains, on top of oracle/adjusted_mclmc.py, oracle/adaptation.da_update and
oracle/diagnostics.effective_sample_size.  Every chain behaves like one jax.vmap lane of the reference.

The kernel being tuned is ``("static", None)`` (adjusted_mclmc: ceil(avg) steps, info.num_integration_steps = avg) or
``("randint" | "uniform" | "fixed", min_steps)`` (adjusted_mclmc_dynamic with that step rule and random_generator_arg in the
state).  The masks are 0 or 1, so m x + (1 - m) y is a select here (exact for finite x, y).
"""
import numpy as np

from . import adjusted_mclmc as ao
from . import prng as oprng
from .adaptation import DAState, da_init, da_update
from .diagnostics import effective_sample_size
from .mclmc_tuning import safediv

F = np.float32
AVG_FLOOR = F(1.1)


def stage_lengths(num_steps, frac_tune1, frac_tune2, frac_tune3, num_windows=1):
    """(n1, n2, n3) after frac /= num_windows (:114-116): int() truncation (:328-330, :445); n3 = 0 when frac_tune3 = 0."""
    f1, f2, f3 = frac_tune1 / num_windows, frac_tune2 / num_windows, frac_tune3 / num_windows
    return int(num_steps * f1), int(num_steps * f2), (int(num_steps * f3) if f3 != 0 else 0)


def num_steps_of(kind, avg, rga):
    """(steps run [C], info.num_integration_steps [C] as float) of the kernel at avg [C] float32."""
    rule, min_steps = kind
    avg = np.asarray(avg, F)
    if rule == "static":
        with np.errstate(invalid="ignore"):
            n = np.where((avg > 0) & np.isfinite(avg), np.ceil(avg), 0).astype(np.int32)
        return n, avg.astype(F)
    if rule == "randint":
        n = ao.steps_randint(rga)
    elif rule == "uniform":
        scale = np.array([ao.rescale(a) for a in avg], F)
        n = np.maximum(np.ceil((oprng.uniform(rga) * scale).astype(F)), min_steps).astype(np.int32)
    else:
        n = np.maximum(np.ceil(avg), max(min_steps, 1)).astype(np.int32)
    return n, n.astype(F)


def transition(kind, keys, state, target, imm, eps, L, coefficients):
    """One kernel call at avg = L / eps (float32): (new state, info, steps, reported steps)."""
    q, logp, g = state[:3]
    rga = state[3] if len(state) > 3 else None
    avg = (np.asarray(L, F) / np.asarray(eps, F)).astype(F)
    n, rep = num_steps_of(kind, avg, rga)
    new, info = ao.adjusted_mclmc_kernel(keys, (q, logp, g), target, imm, eps, n, coefficients)
    if rga is not None:
        new = (*new, oprng.split(rga, 2)[:, 1])
    return new, info, n, rep


def da_update_masked(da, acceptance_rate, target, mask):
    """update_da then with_mask on all five fields (:267-277); da = (log_step, log_step_avg, step, avg_error, mu) [C]."""
    up = DAState(*(np.asarray(x, F) for x in da_update(DAState(*da), acceptance_rate, target=target)))
    up = up._replace(step=np.asarray(up.step, F))
    m = np.asarray(mask, bool)
    return tuple(np.where(m, u, F(o)).astype(F) for u, o in zip(up, da))


def clamp_step(log_step, L):
    """step = lax.clamp(1e-5, exp(log_step), L / 1.1) and the log round trip (:279-282): (step, log step)."""
    with np.errstate(over="ignore"):
        step = np.minimum(np.maximum(np.exp(np.asarray(log_step, F)).astype(F), F(1e-5)), (np.asarray(L, F) / AVG_FLOOR)
                          .astype(F)).astype(F)
    return step, np.log(step).astype(F)


def moments_update(x, total, moments, weight, zero_prevention):
    """incremental_value_update(expectation=(x, x^2), weight, zero_prevention) (util.py:291-319): (total, moments)."""
    exp = np.stack([x, (x * x).astype(F)], axis=1)
    num = ((total[:, None, None] * moments).astype(F) + (weight[:, None, None] * exp).astype(F)).astype(F)
    den = ((total + weight).astype(F) + zero_prevention).astype(F)
    return (total + weight).astype(F), safediv(num, den[:, None, None])


def handle_nans(previous, new):
    """:494-507 on the state: (nonans [C], state).  A non-finite position reverts the whole state, else nan_to_num."""
    nonans = np.all(np.isfinite(new[0]), axis=1)
    out = []
    for a, b in zip(new, previous):
        a = np.nan_to_num(a) if a.dtype.kind == "f" else a
        nm = nonans.reshape((-1,) + (1,) * (a.ndim - 1))
        out.append(np.where(nm, a, b).astype(a.dtype))
    return nonans, tuple(out)


def tune_step(kind, keys, state, target, imm, eps, L, da, streaming, mask, fix_L, tgt_acc, coefficients, info=None):
    """One dual_avg_step (:236-311) for per-chain step keys [C, 2].  da: five [C] arrays; streaming (total [C], moments
    [C, 2, D]).  info (optional) = (new state, info, steps, reported) of a transition already run (teacher forcing).
    Returns (state, eps, L, da, streaming, nonans, steps, reported)."""
    eps, L = np.asarray(eps, F), np.asarray(L, F)
    C = eps.shape[0]
    new, inf, n, rep = info if info is not None else transition(kind, keys, state, target, imm, eps, L, coefficients)
    nonans, st = handle_nans(state, new)
    m = np.broadcast_to(np.asarray(mask, F), (C,))
    da = da_update_masked(da, inf.acceptance_rate, tgt_acc, m == 1)
    step, log_step = clamp_step(da[0], L)
    da = (log_step,) + tuple(da[1:])
    weight = ((F(1) - m) * nonans.astype(F) * step).astype(F)
    streaming = moments_update(st[0], streaming[0], streaming[1], weight, m)
    new_eps = np.where(m == 1, step, eps).astype(F)
    new_L = L if fix_L else np.where(m == 1, (L * (step / eps).astype(F)).astype(F), L).astype(F)
    return st, new_eps, new_L, da, streaming, nonans, n, rep


def _pass(kind, base, n, n_masked, state, target, imm, eps, L, fix_L, tgt_acc, coefficients, count):
    """step_size_adaptation (:315-325) with a fresh DA, then step_size = final_da (:368-369, :432)."""
    C, D = state[0].shape
    d = da_init(eps)
    da = tuple(np.broadcast_to(np.asarray(x, F), (C,)).copy() for x in d)
    streaming = (np.zeros(C, F), np.zeros((C, 2, D), F))
    for t in range(n):
        keys = oprng.fold_in(base, t)
        state, eps, L, da, streaming, _, _, rep = tune_step(kind, keys, state, target, imm, eps, L, da, streaming,
                                                            float(t < n_masked), fix_L, tgt_acc, coefficients)
        count = (count + rep).astype(F)
    eps = np.exp(da[1]).astype(F)
    return state, eps, L, streaming, count


def window(kind, key, n1, n2, state, target, imm, eps, L, tgt_acc, coefficients, diagonal_preconditioning, max_,
           tuning_factor, target_k, count):
    """adjusted_mclmc_make_L_step_size_adaptation(...)(state, params, num_steps, key) (:327-434)."""
    rk = oprng.split(key, 2)[:, 1]
    p = oprng.split(rk, 2)
    state, eps, L, (_, mom), count = _pass(kind, p[:, 0], n1 + n2, n1, state, target, imm, eps, L, True, tgt_acc,
                                           coefficients, count)
    if n2 != 0:
        var = (mom[:, 1] - (mom[:, 0] * mom[:, 0]).astype(F)).astype(F)
        D = var.shape[1]
        if max_ == "max":
            contract = (np.sqrt((var.max(axis=1) * F(D)).astype(F)) * F(tuning_factor)).astype(F)
        else:
            contract = (np.sqrt(var.sum(axis=1, dtype=F)) * F(tuning_factor)).astype(F)
        with np.errstate(invalid="ignore", divide="ignore"):
            change = np.clip((contract / L).astype(F), F(0), F(2)).astype(F)
        L = (L * change).astype(F)
        eps = (eps * change).astype(F)
        if diagonal_preconditioning:
            imm = var
        L = (F(target_k) * eps).astype(F)
        state, eps, L, _, count = _pass(kind, p[:, 1], n1, n1, state, target, imm, eps, L, False, tgt_acc, coefficients,
                                        count)
    return state, eps, L, imm, count


def ess_L(hist, L, max_, l_factor=0.5):
    """adaptation_L's L update (:465-486) from the position history [n3, C, D]."""
    n3, C, _ = hist.shape
    ess = np.stack([np.atleast_1d(effective_sample_size(hist[:, c][None], chain_axis=0, sample_axis=1))
                    for c in range(C)]).astype(F)
    r = (ess.min(axis=1) if max_ == "max" else ess.mean(axis=1, dtype=F)).astype(F)
    r = (r / F(n3)).astype(F)
    with np.errstate(divide="ignore"):
        return np.minimum(((F(l_factor) * L).astype(F) / r).astype(F), (L * F(2.0)).astype(F)).astype(F)


def find_L_and_step_size(kind, chain_keys, num_steps, state, target, coefficients, tgt_acc, frac_tune1=0.1,
                         frac_tune2=0.1, frac_tune3=0.0, diagonal_preconditioning=True, params=None, max_="avg",
                         num_windows=1, tuning_factor=1.3, target_num_integration_steps=2.0):
    """adjusted_mclmc_find_L_and_step_size (:26-205) for every chain: chain_keys [C, 2] are the chains' own keys.  params =
    (L, step_size, inverse_mass_matrix) broadcastable to [C], [C], [C, D].  Returns (state, (L, eps, imm), count [C])."""
    state = tuple(np.asarray(x) for x in state)
    C, D = state[0].shape
    n1, n2, n3 = stage_lengths(num_steps, frac_tune1, frac_tune2, frac_tune3, num_windows)
    if params is None:
        s = np.sqrt(F(D)).astype(F)
        params = (s, (s * F(0.2)).astype(F), F(1))
    eps = np.broadcast_to(np.asarray(params[1], F), (C,)).copy()
    imm = np.broadcast_to(np.asarray(params[2], F), (C, D)).copy()
    tk = F(target_num_integration_steps)
    L = (tk * eps).astype(F)
    parts = oprng.split(chain_keys, 2)
    part1, part2 = parts[:, 0], parts[:, 1]
    count = np.zeros(C, F)
    for i in range(num_windows):
        state, eps, L, imm, count = window(kind, oprng.fold_in(part1, i), n1, n2, state, target, imm, eps, L, tgt_acc,
                                           coefficients, diagonal_preconditioning, max_, tuning_factor, tk, count)
    if n3 != 0:
        for i in range(num_windows):
            part2 = oprng.fold_in(part2, i)
            k = oprng.split(part2, 2)
            hist = []
            for t in range(n3):
                state, _, _, rep = transition(kind, oprng.fold_in(k[:, 0], t), state, target, imm, eps, L, coefficients)
                count = (count + rep).astype(F)
                hist.append(state[0])
            L = ess_L(np.stack(hist), L, max_)
            state, eps, L, imm, count = window(kind, k[:, 1], n1, 0, state, target, imm, eps, L, tgt_acc, coefficients,
                                               diagonal_preconditioning, max_, tuning_factor, None, count)
    L = (tk * eps).astype(F)
    return state, (L, eps, imm), count
