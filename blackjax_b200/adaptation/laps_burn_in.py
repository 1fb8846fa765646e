"""Step-level pieces of LAPS (blackjax/adaptation/laps_burn_in.py, laps.py, eca.py) on the device, for callers that drive the
phases themselves and for tests.  ``laps.laps`` strings them together.

All functions work in place on an engine's chains and one LAPS state buffer ``adap`` (float32, libbjx
``bjx_laps_state_floats``).  ``phase_key`` is one raw key ``uint32 [2]`` (a torch tensor on any device, or a numpy array):
chain c at step t uses ``split(split(phase_key)[0], (N, T))[c, t]``.
"""
import ctypes as C

import numpy as np
import torch

from .._lib import LapsBurnInConfig, check, lib, ptr

__all__ = ["BURN_IN_INFO", "ADJUSTED_INFO", "new_state", "header", "inverse_mass_matrix", "history", "initialize",
           "burn_in_step_", "burn_in_run_", "switch_", "adjusted_step_", "adjusted_run_"]

# fields of the info rows the device writes
BURN_IN_INFO = ("L", "step_size", "EEVPD_wanted", "EEVPD", "equi_diag", "equi_full", "r_max", "r_avg", "entropy")
ADJUSTED_INFO = ("L", "step_size", "acc_prob", "equi_diag")
_HDR = 16
LS_L, LS_EPS, LS_COUNT, LS_STOP, LS_EEVPD, LS_EEVPD_W, LS_EQUI_FULL, LS_LO, LS_HI, LS_TERM = range(10)


def _key(phase_key):
    k = phase_key.detach().cpu().numpy() if isinstance(phase_key, torch.Tensor) else np.asarray(phase_key)
    k = k.astype(np.int64).reshape(-1) & 0xFFFFFFFF
    if k.shape != (2,):
        raise ValueError("phase_key must be one raw key of 2 uint32 words")
    return (C.c_uint32 * 2)(int(k[0]), int(k[1]))


def config(save_num, alpha=1.9, C_=0.1, r_end=0.01, bias_type=3, early_stop=True, equi_full=True):
    return LapsBurnInConfig(int(save_num), float(alpha), float(C_), float(r_end), int(bias_type), int(bool(early_stop)),
                            int(bool(equi_full)))


def new_state(eng, save_num, equi_full=True):
    n = lib().bjx_laps_state_floats(eng.C, eng.D, int(save_num), int(bool(equi_full)))
    if n < 0:
        raise ValueError("save_num = rint(save_frac * num_steps1) must be at least 1")
    return torch.zeros(int(n), dtype=torch.float32, device=eng.device)


def header(adap):
    """The adaptation state's scalars: L, step_size, step_count, stopped, EEVPD, EEVPD_wanted, equi_full and the
    bisection's (lower, upper, terminated)."""
    h = adap[:_HDR].cpu()
    i = h.view(torch.int32)
    return {"L": float(h[LS_L]), "step_size": float(h[LS_EPS]), "step_count": int(i[LS_COUNT]),
            "stopped": bool(i[LS_STOP]), "EEVPD": float(h[LS_EEVPD]), "EEVPD_wanted": float(h[LS_EEVPD_W]),
            "equi_full": float(h[LS_EQUI_FULL]), "bounds": (float(h[LS_LO]), float(h[LS_HI])),
            "terminated": bool(h[LS_TERM] != 0)}


def inverse_mass_matrix(adap, D):
    """A view of the state's M^-1 [D]."""
    return adap[_HDR:_HDR + D]


def _up4(n):
    return (n + 3) & ~3


def history(adap, D, save_num):
    """The history ring [save_num, D] (slot t % save_num holds step t's ensemble mean of x)."""
    o = _HDR + _up4(D)
    return adap[o:o + save_num * D].view(save_num, D)


def initialize(eng, q, adap, save_num):
    """laps_burn_in.initialize after sample_init, and the burn-in's initial adaptation state.  Returns (q, u, logp, g)."""
    q = q.contiguous().clone()
    logp = torch.empty(eng.C, dtype=torch.float32, device=eng.device)
    g, u = torch.empty_like(q), torch.empty_like(q)
    eng.ensure_metric(torch.ones(eng.D, dtype=torch.float32, device=eng.device), diagonal_only=True)
    check(lib().bjx_laps_init(eng.h, ptr(q), ptr(logp), ptr(g), ptr(u), ptr(adap), int(save_num)), eng.h)
    return q, u, logp, g


def burn_in_step_(eng, phase_key, t, num_steps, state, adap, cfg, info=None):
    """Burn-in step t in place; state = (q, u, logp, g); info (optional) [num_steps, 9] float32 on the device."""
    q, u, logp, g = state
    check(lib().bjx_laps_burn_in_step(eng.h, _key(phase_key), int(t), int(num_steps), ptr(q), ptr(u), ptr(logp), ptr(g),
                                      ptr(adap), C.byref(cfg), ptr(info)), eng.h)


def burn_in_run_(eng, phase_key, num_steps, state, adap, cfg, info=None, chunk=64):
    """Every burn-in step, the stop flag read once per ``chunk`` steps.  Returns the number of steps taken."""
    q, u, logp, g = state
    n = C.c_int32()
    check(lib().bjx_laps_burn_in_run(eng.h, _key(phase_key), int(num_steps), ptr(q), ptr(u), ptr(logp), ptr(g), ptr(adap),
                                     C.byref(cfg), ptr(info), int(chunk), C.byref(n)), eng.h)
    return n.value


def switch_(eng, adap, diagonal_preconditioning):
    """laps.py:250-257 on the state; installs the adjusted phase's metric on the engine.  Returns it."""
    check(lib().bjx_laps_switch(eng.h, ptr(adap), int(bool(diagonal_preconditioning))), eng.h)
    imm = (inverse_mass_matrix(adap, eng.D) if diagonal_preconditioning
           else torch.ones(eng.D, dtype=torch.float32, device=eng.device))
    eng.set_metric(imm, diagonal_only=True)
    eng._imm_key = None
    return imm


def adjusted_step_(eng, phase_key, t, num_samples, state, adap, save_num, steps_per_sample, target, diagnostics=True,
                   info=None):
    """Adjusted step t in place; state = (q, logp, g); info (optional) [num_samples, 4]."""
    q, logp, g = state
    check(lib().bjx_laps_adjusted_step(eng.h, _key(phase_key), int(t), int(num_samples), ptr(q), ptr(logp), ptr(g),
                                       ptr(adap), int(save_num), int(steps_per_sample), float(target),
                                       int(bool(diagnostics)), ptr(info)), eng.h)


def adjusted_run_(eng, phase_key, num_samples, state, adap, save_num, steps_per_sample, target, diagnostics=True,
                  info=None):
    q, logp, g = state
    check(lib().bjx_laps_adjusted_run(eng.h, _key(phase_key), int(num_samples), ptr(q), ptr(logp), ptr(g), ptr(adap),
                                      int(save_num), int(steps_per_sample), float(target), int(bool(diagnostics)),
                                      ptr(info)), eng.h)
