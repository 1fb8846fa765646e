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


def _rank_call(history, logdensity_fn, max_scratch_bytes):
    """(engine, contiguous history, T, C, D, scratch) for the rank-normalised diagnostics: the scratch of the widest pass
    over the dimensions that fits max_scratch_bytes, as bjx_rank_diagnostics picks it from the buffer it is given.  When
    not even one dimension fits, the library rejects the call and names the bytes it needs."""
    from ._engine import get_engine
    if history.ndim != 3:
        raise ValueError("history must have shape [num_samples, n_chains, dim]")
    T, C, D = history.shape
    history = history.contiguous()
    eng = get_engine(history[0], logdensity_fn)
    need = lambda dc: int(lib().bjx_rank_diagnostics_scratch_bytes(int(T), int(C), int(D), int(dc)))  # noqa: E731
    lo, hi = 0, D
    if T >= 4:
        while lo < hi:
            mid = lo + (hi - lo + 1) // 2
            if 0 <= need(mid) <= max_scratch_bytes:
                lo = mid
            else:
                hi = mid - 1
    if 32 <= lo < D:
        lo -= lo % 32
    nbytes = need(lo) if lo > 0 else 256
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=history.device)
    return eng, history, T, C, D, scratch


def rank_normalize(history, logdensity_fn, folded=False, max_scratch_bytes=1 << 31):
    """``blackjax.diagnostics._rank_normalize`` (blackjax/diagnostics.py:367-401) applied to the split chains of
    ``history`` [num_samples, n_chains, dim]: each chain's two halves of h = num_samples // 2 draws (an odd last draw is
    dropped) become 2 * n_chains chains, and every dimension's pooled draws are replaced by their Blom scores
    Phi^-1((r - 3/8) / (n + 1/4)), ties ranked by pooled index.  ``folded=True`` scores |x - median| instead (the tail
    component of ``rhat``).  Returns [h, 2 * n_chains, dim], split chain C + c holding the second half of chain c.
    ``logdensity_fn`` only selects the engine."""
    eng, history, T, C, D, scratch = _rank_call(history, logdensity_fn, max_scratch_bytes)
    out = torch.empty(T // 2, 2 * C, D, dtype=torch.float32, device=history.device)
    check(lib().bjx_rank_normalize(eng.h, ptr(history), int(T), int(bool(folded)), ptr(out), ptr(scratch),
                                   scratch.numel()), eng.h)
    return out


def _rank_diagnostics(history, logdensity_fn, max_scratch_bytes, prob=0.90, rhat=False, bulk=False, tail=False):
    eng, history, T, C, D, scratch = _rank_call(history, logdensity_fn, max_scratch_bytes)
    out = [torch.empty(D, dtype=torch.float32, device=history.device) if want else None for want in (rhat, bulk, tail)]
    check(lib().bjx_rank_diagnostics(eng.h, ptr(history), int(T), float(prob), *(ptr(o) for o in out), ptr(scratch),
                                     scratch.numel()), eng.h)
    return [o for o in out if o is not None][0]


def rhat(history, logdensity_fn, max_scratch_bytes=1 << 31):
    """``blackjax.rhat`` (blackjax/diagnostics.py:92-155), the rank-normalised split-R-hat of Vehtari et al. (2021), for
    ``history`` [num_samples, n_chains, dim]: per dimension the larger of the split R-hat of the rank-normalised draws
    and that of the rank-normalised folded draws |x - median|.  Needs num_samples >= 4; one chain is allowed (its two
    halves are compared).  A dimension with a NaN draw reports NaN.  ``max_scratch_bytes`` bounds the device scratch:
    dimensions are processed as many at a time as fit.  ``logdensity_fn`` only selects the engine."""
    return _rank_diagnostics(history, logdensity_fn, max_scratch_bytes, rhat=True)


def ess_bulk(history, logdensity_fn, max_scratch_bytes=1 << 31):
    """``blackjax.ess_bulk`` (blackjax/diagnostics.py:404-444): ``effective_sample_size`` of the rank-normalised split
    chains of ``history`` [num_samples, n_chains, dim], per dimension.  NaN for a dimension with a NaN draw."""
    return _rank_diagnostics(history, logdensity_fn, max_scratch_bytes, bulk=True)


def ess_tail(history, logdensity_fn, prob=0.90, max_scratch_bytes=1 << 31):
    """``blackjax.ess_tail`` (blackjax/diagnostics.py:447-522): the smaller of the ESS of the split-chain indicators
    1[x <= q_lo] and 1[x >= q_hi], with q_lo, q_hi the pooled linear quantiles at (1 - prob) / 2 and (1 + prob) / 2.
    NaN for a dimension with a NaN draw."""
    return _rank_diagnostics(history, logdensity_fn, max_scratch_bytes, prob=prob, tail=True)
