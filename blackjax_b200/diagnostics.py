"""Diagnostics on device-resident draws (SURVEY.md section 8f item 3)."""
import torch

from ._lib import check, lib, ptr


def potential_scale_reduction(history, logdensity_fn):
    """``blackjax.diagnostics.potential_scale_reduction`` (blackjax/diagnostics.py:39-89) for ``history`` of shape
    [num_samples, n_chains, dim] (the layout ``sample_hmc_native`` / ``bjx_hmc_sample`` writes): R-hat per dimension.
    ``logdensity_fn`` only selects the engine (device, shape)."""
    from ._engine import get_engine
    if history.ndim != 3:
        raise ValueError("history must have shape [num_samples, n_chains, dim]")
    T, C, D = history.shape
    assert C > 1, "potential_scale_reduction as implemented only works for two or more chains."
    history = history.contiguous()
    eng = get_engine(history[0], logdensity_fn)
    rhat = torch.empty(D, dtype=torch.float32, device=history.device)
    scratch = torch.empty(2 * C * D + 4 + 4 * D, dtype=torch.float32, device=history.device)
    check(lib().bjx_potential_scale_reduction(eng.h, ptr(history), int(T), ptr(rhat), ptr(scratch)), eng.h)
    return rhat


def effective_sample_size(history, logdensity_fn, per_chain=False):
    """``blackjax.diagnostics.effective_sample_size`` (blackjax/diagnostics.py:159-305) for ``history`` of shape
    [num_samples, n_chains, dim]: ESS per dimension (Geyer's initial positive / monotone sequence estimators on the
    chain-averaged autocovariance, evaluated on the device).  ``logdensity_fn`` only selects the engine.

    ``per_chain=True``: the single-chain ESS of every chain, ``effective_sample_size(history[:, c, None, :])`` for each
    c, as an [n_chains, dim] tensor (the estimate MCLMC's tuner uses)."""
    from ._engine import get_engine
    if history.ndim != 3:
        raise ValueError("history must have shape [num_samples, n_chains, dim]")
    T, C, D = history.shape
    assert T > 1, f"The input array must have at least 2 samples, got only {T}."
    history = history.contiguous()
    eng = get_engine(history[0], logdensity_fn)
    if per_chain:
        ess = torch.empty(C, D, dtype=torch.float32, device=history.device)
        check(lib().bjx_mclmc_ess_per_chain(eng.h, ptr(history), int(T), ptr(ess), None), eng.h)
        return ess
    ess = torch.empty(D, dtype=torch.float32, device=history.device)
    n = int(lib().bjx_ess_scratch_floats(int(T), int(C), int(D)))
    scratch = torch.empty((n + 1) // 2, dtype=torch.float64, device=history.device).view(torch.float32)
    check(lib().bjx_effective_sample_size(eng.h, ptr(history), int(T), ptr(ess), ptr(scratch)), eng.h)
    return ess
