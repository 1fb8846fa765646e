"""Driver loop mirroring ``blackjax.util.run_inference_algorithm`` (blackjax/util.py:150-213)."""
import torch

from . import random as bjx_random


def _native_run(name, rng_key, eng, q, num_steps, thin, keep_history, chain_offset, *stats):
    """What every ``sample_*_native`` shares once the engine is set up: the one step key on the device (shared step-key
    mode from ``chain_offset``), the history [num_steps // thin, C, D] or None, and one [num_steps, C] array per dtype in
    ``stats``.  Returns (key, history, *stats)."""
    key = rng_key.to(q.device).contiguous()
    if key.ndim != 1:
        raise ValueError(f"sample_{name}_native takes ONE rng_key of shape [2]")
    eng._key_mode(key, chain_offset)
    C, D = q.shape
    hist = torch.empty(num_steps // thin, C, D, dtype=torch.float32, device=q.device) if keep_history else None
    return (key, hist, *(torch.empty(num_steps, C, dtype=dt, device=q.device) for dt in stats))


def sample_hmc_native(rng_key, state, logdensity_fn, step_size, inverse_mass_matrix, num_integration_steps, num_steps,
                      *, multinomial=False, thin=1, keep_history=True, chain_offset=0):
    """``run_inference_algorithm`` for HMC / multinomial HMC without a Python-level loop: libbjx ``bjx_hmc_sample``
    derives ``split(rng_key, num_steps)`` on the device and enqueues every transition back to back (no host sync), so
    small problems run at kernel-launch rate.  Same draws as ``num_steps`` calls of ``hmc.step(split(rng_key, T)[t], .)``.
    Returns (final HMCState, positions [num_steps // thin, C, D] or None, acceptance rates [num_steps, C])."""
    from ._engine import get_engine
    from ._lib import check, lib, ptr
    from .mcmc.hmc import HMCState
    q, logp, g = (t.clone() for t in state)
    eng = get_engine(q, logdensity_fn)
    eng.ensure_metric(inverse_mass_matrix)
    key, hist, acc = _native_run("hmc", rng_key, eng, q, num_steps, thin, keep_history, chain_offset, torch.float32)
    eps, eps_dev = eng._eps(step_size)
    check(lib().bjx_hmc_sample(eng.h, ptr(key), ptr(q), ptr(logp), ptr(g), eps, ptr(eps_dev), int(num_integration_steps),
                               int(num_steps), int(bool(multinomial)), ptr(hist), int(thin), ptr(acc)), eng.h)
    return HMCState(q, logp, g), hist, acc


def sample_nuts_native(rng_key, state, logdensity_fn, step_size, inverse_mass_matrix, num_steps, *, max_num_doublings=10,
                       thin=1, keep_history=True, chain_offset=0):
    """``run_inference_algorithm`` for NUTS without a Python-level loop (libbjx ``bjx_nuts_sample``): same draws as
    ``num_steps`` calls of ``nuts.step(split(rng_key, T)[t], .)``.  Returns (final HMCState, positions
    [num_steps // thin, C, D] or None, acceptance rates [num_steps, C], tree sizes int32 [num_steps, C])."""
    from ._engine import get_engine
    from ._lib import check, lib, ptr
    from .mcmc.hmc import HMCState
    q, logp, g = (t.clone() for t in state)
    eng = get_engine(q, logdensity_fn, max_tree_depth=max(10, max_num_doublings))
    eng.ensure_metric(inverse_mass_matrix)
    key, hist, acc, n_int = _native_run("nuts", rng_key, eng, q, num_steps, thin, keep_history, chain_offset,
                                        torch.float32, torch.int32)
    eps, eps_dev = eng._eps(step_size)
    check(lib().bjx_nuts_sample(eng.h, ptr(key), ptr(q), ptr(logp), ptr(g), eps, ptr(eps_dev), int(max_num_doublings),
                                int(num_steps), ptr(hist), int(thin), ptr(acc), ptr(n_int)), eng.h)
    return HMCState(q, logp, g), hist, acc, n_int


def sample_mclmc_native(rng_key, state, logdensity_fn, L, step_size, num_steps, *, inverse_mass_matrix=1.0,
                        integrator="isokinetic_mclachlan", desired_energy_var_max_ratio=float("inf"),
                        desired_energy_var=5e-4, thin=1, keep_history=True, chain_offset=0):
    """``run_inference_algorithm`` for MCLMC without a Python-level loop (libbjx ``bjx_mclmc_sample``): same draws as
    ``num_steps`` calls of ``mclmc.step(split(rng_key, T)[t], .)``.  Returns (final IntegratorState, positions
    [num_steps // thin, C, D] or None, energy changes [num_steps, C])."""
    from ._engine import get_engine
    from ._lib import check, lib, ptr
    from .mcmc import integrators
    from .mcmc.hmc import IntegratorState
    from .mcmc.mclmc import energy_cutoff, metric_tensor
    q, p, logp, g = (t.clone() for t in state)
    eng = get_engine(q, logdensity_fn)
    eng.set_integrator(integrators.as_coefficients(integrator))
    eng.ensure_metric(metric_tensor(eng, inverse_mass_matrix), diagonal_only=True)
    key, hist, de = _native_run("mclmc", rng_key, eng, q, num_steps, thin, keep_history, chain_offset, torch.float32)
    eps, eps_dev = eng._eps(step_size)
    L, L_dev = eng._eps(L, "L")
    check(lib().bjx_mclmc_sample(eng.h, ptr(key), ptr(q), ptr(p), ptr(logp), ptr(g), eps, ptr(eps_dev), L, ptr(L_dev),
                                 energy_cutoff(q.shape[1], desired_energy_var_max_ratio, desired_energy_var),
                                 int(num_steps), ptr(hist), int(thin), ptr(de)), eng.h)
    return IntegratorState(q, p, logp, g), hist, de


def sample_adjusted_mclmc_native(rng_key, state, logdensity_fn, step_size, num_steps, *, num_integration_steps=None,
                                 integration_steps_fn=None, integration_steps_params=(), L_proposal_factor=float("inf"),
                                 inverse_mass_matrix=1.0, integrator="isokinetic_mclachlan", divergence_threshold=1000,
                                 thin=1, keep_history=True, chain_offset=0):
    """``run_inference_algorithm`` for adjusted MCLMC without a Python-level loop (libbjx ``bjx_adjusted_mclmc_sample``):
    same draws as ``num_steps`` calls of the step API with keys ``split(rng_key, T)[t]``.

    Static (``adjusted_mclmc``): ``state`` is an HMCState and ``num_integration_steps`` an int.  Dynamic
    (``adjusted_mclmc_dynamic``): ``state`` is a DynamicHMCState and ``integration_steps_fn`` one of the rules evaluated on
    the device -- the default ``randint(key, (), 1, 10)`` or ``make_random_trajectory_length_fn(...)`` with
    ``integration_steps_params = (avg_num_integration_steps,)``; ``random_generator_arg`` advances to ``split(key)[1]`` per
    transition.  Other step-count functions go through the step API.  Returns (final state, positions
    [num_steps // thin, C, D] or None, acceptance rates [num_steps, C], step counts int32 [num_steps, C])."""
    from ._engine import get_engine
    from ._lib import AMCLMC_STEPS_FIXED, AMCLMC_STEPS_RANDINT, AMCLMC_STEPS_UNIFORM, check, lib, ptr
    from .mcmc import adjusted_mclmc_dynamic, integrators
    from .mcmc.dynamic_hmc import DynamicHMCState
    from .mcmc.hmc import HMCState
    from .mcmc.mclmc import metric_tensor
    dynamic = isinstance(state, DynamicHMCState)
    rule, min_steps, n, scale, rga = AMCLMC_STEPS_FIXED, 0, 0, 0.0, None
    avg_dev = None  # a per-chain average trajectory length [C], evaluated by the kernel chain by chain
    if dynamic:
        fn = integration_steps_fn or adjusted_mclmc_dynamic._integration_steps
        if getattr(fn, "device_rule", None) is None:
            raise ValueError("sample_adjusted_mclmc_native evaluates the default randint rule and "
                             "make_random_trajectory_length_fn(...) on the device; use the step API for other "
                             "integration_steps_fn")
        rule, min_steps = fn.device_rule
        if rule != AMCLMC_STEPS_RANDINT and adjusted_mclmc_dynamic._per_chain(integration_steps_params):
            avg_dev = integration_steps_params[0].to(state[0].device, torch.float32).contiguous()
            if rule == AMCLMC_STEPS_FIXED:
                min_steps = max(int(min_steps), 1)  # max(ceil(avg), 1)
        elif rule == AMCLMC_STEPS_FIXED:
            n = fn(None, *integration_steps_params)
        elif rule == AMCLMC_STEPS_UNIFORM:
            (avg,) = integration_steps_params
            scale = float(adjusted_mclmc_dynamic.rescale(avg))
        q, logp, g, rga = (t.clone() for t in state)
        if rga.dtype not in (torch.uint32, torch.int32) or tuple(rga.shape) != (q.shape[0], 2):
            raise ValueError("random_generator_arg must be uint32 [n_chains, 2]")
        rga = rga.contiguous()
    else:
        if num_integration_steps is None:
            raise ValueError("the static sampler needs num_integration_steps")
        from .mcmc.adjusted_mclmc import steps_argument
        n = steps_argument(num_integration_steps)
        if isinstance(n, torch.Tensor):
            if not n.is_floating_point():
                raise ValueError("the native loop takes an int or a float per-chain num_integration_steps")
            avg_dev, n = n.to(state[0].device, torch.float32).contiguous(), 0
        q, logp, g = (t.clone() for t in state)
    eng = get_engine(q, logdensity_fn, divergence_threshold=divergence_threshold)
    eng.set_integrator(integrators.as_coefficients(integrator))
    eng.ensure_metric(metric_tensor(eng, inverse_mass_matrix), diagonal_only=True)
    key, hist, acc, steps = _native_run("adjusted_mclmc", rng_key, eng, q, num_steps, thin, keep_history, chain_offset,
                                        torch.float32, torch.int32)
    eps, eps_dev = eng._eps(step_size)
    C = q.shape[0]
    if avg_dev is not None and tuple(avg_dev.shape) != (C,):
        raise ValueError(f"per-chain average trajectory lengths must have shape ({C},)")
    check(lib().bjx_set_integration_steps_avg(eng.h, ptr(avg_dev)), eng.h)
    try:
        check(lib().bjx_adjusted_mclmc_sample(eng.h, ptr(key), ptr(q), ptr(logp), ptr(g), eps, ptr(eps_dev),
                                              float(L_proposal_factor), int(rule), int(n), scale, int(min_steps),
                                              ptr(rga), int(num_steps), ptr(hist), int(thin), ptr(acc), ptr(steps)),
              eng.h)
    finally:
        if avg_dev is not None:
            check(lib().bjx_set_integration_steps_avg(eng.h, None), eng.h)
            eng._avg_keepalive = avg_dev  # the launches are asynchronous
    final = DynamicHMCState(q, logp, g, rga) if dynamic else HMCState(q, logp, g)
    return final, hist, acc, steps


def sample_gist_native(rng_key, state, logdensity_fn, step_size, inverse_mass_matrix, num_steps, *,
                       instance="trajectory_length", path_fraction=0.5, max_num_steps=1024, num_integration_steps=1,
                       criterion="symmetric", max_search_steps=10, integrator=None, divergence_threshold=1000, thin=1,
                       keep_history=True, chain_offset=0):
    """``run_inference_algorithm`` for GIST without a Python-level loop (libbjx ``bjx_gist_sample``): one persistent
    launch, same draws as ``num_steps`` calls of ``gist_trajectory_length`` (``instance="trajectory_length"``) or
    ``gist_step_size`` (``instance="step_size"``, ``step_size`` being the initial step size) with the step keys
    ``split(rng_key, T)[t]``.  Returns (final GISTState, positions [num_steps // thin, C, D] or None, acceptance rates
    [num_steps, C], num_integration_steps int32 [num_steps, C])."""
    from ._engine import get_engine
    from ._lib import check, lib, ptr
    from .mcmc import integrators
    from .mcmc.composed import _seam, step_size as ss, trajectory_length as tl
    if instance == "trajectory_length":
        tuning = tl.tuning(path_fraction, max_num_steps)
    elif instance == "step_size":
        tuning = ss.tuning(num_integration_steps, criterion, max_search_steps)
    else:
        raise ValueError(f"instance must be 'trajectory_length' or 'step_size', got {instance!r}")
    q, logp, g = (t.clone() for t in state)
    eng = get_engine(q, logdensity_fn, divergence_threshold=divergence_threshold)
    eng.set_integrator(integrators.as_coefficients(integrator or integrators.velocity_verlet))
    eng.ensure_metric(inverse_mass_matrix)
    key, hist, acc, n_int = _native_run("gist", rng_key, eng, q, num_steps, thin, keep_history, chain_offset,
                                        torch.float32, torch.int32)
    eps, eps_dev = eng._eps(step_size)
    check(lib().bjx_gist_sample(eng.h, tuning.params, ptr(key), ptr(q), ptr(logp), ptr(g), eps, ptr(eps_dev),
                                int(num_steps), ptr(hist), int(thin), ptr(acc), ptr(n_int)), eng.h)
    return _seam.GISTState(q, logp, g), hist, acc, n_int


def _sample_langevin_native(sampler, rng_key, state, logdensity_fn, step_size, num_steps, thin, keep_history,
                            chain_offset, inverse_mass_matrix=None):
    from ._engine import get_engine
    from ._lib import check, lib, ptr
    q, logp, g = (t.clone() for t in state)
    eng = get_engine(q, logdensity_fn)
    fn = lib().bjx_mala_sample
    if sampler == "barker":
        from .mcmc import barker
        barker.install_metric(eng, inverse_mass_matrix)
        fn = lib().bjx_barker_sample
    key, hist, acc = _native_run(sampler, rng_key, eng, q, num_steps, thin, keep_history, chain_offset, torch.float32)
    eps, eps_dev = eng._eps(step_size)
    check(fn(eng.h, ptr(key), ptr(q), ptr(logp), ptr(g), eps, ptr(eps_dev), int(num_steps), ptr(hist), int(thin),
             ptr(acc)), eng.h)
    return (q, logp, g), hist, acc


def sample_mala_native(rng_key, state, logdensity_fn, step_size, num_steps, *, thin=1, keep_history=True,
                       chain_offset=0):
    """``run_inference_algorithm`` for MALA without a Python-level loop (libbjx ``bjx_mala_sample``): the same draws as
    ``num_steps`` calls of ``mala`` with the step keys ``split(rng_key, T)[t]``.  Returns (final MALAState, positions
    [num_steps // thin, C, D] or None, acceptance rates [num_steps, C])."""
    from .mcmc.mala import MALAState
    final, hist, acc = _sample_langevin_native("mala", rng_key, state, logdensity_fn, step_size, num_steps, thin,
                                               keep_history, chain_offset)
    return MALAState(*final), hist, acc


def sample_barker_native(rng_key, state, logdensity_fn, step_size, num_steps, inverse_mass_matrix=None, *, thin=1,
                         keep_history=True, chain_offset=0):
    """``run_inference_algorithm`` for Barker's proposal without a Python-level loop (libbjx ``bjx_barker_sample``), as
    ``sample_mala_native``; ``inverse_mass_matrix=None`` means ones."""
    from .mcmc.barker import BarkerState
    final, hist, acc = _sample_langevin_native("barker", rng_key, state, logdensity_fn, step_size, num_steps, thin,
                                               keep_history, chain_offset, inverse_mass_matrix)
    return BarkerState(*final), hist, acc


def sample_elliptical_slice_native(rng_key, state, loglikelihood_fn, mean, cov, num_steps, *, max_subiter=1000, thin=1,
                                   keep_history=True, chain_offset=0):
    """``run_inference_algorithm`` for elliptical slice sampling without a Python-level loop (libbjx
    ``bjx_elliptical_slice_sample``): the same draws as ``num_steps`` calls of ``elliptical_slice`` with the step keys
    ``split(rng_key, T)[t]``.  Returns (final EllipSliceState, positions [num_steps // thin, C, D] or None, subiter
    int32 [num_steps, C])."""
    from ._engine import get_engine
    from ._lib import check, lib, ptr
    from .mcmc.elliptical_slice import EllipSliceState, _check_cov
    _check_cov(cov)
    q, logl = (t.clone() for t in state)
    eng = get_engine(q, loglikelihood_fn)
    eng.ensure_elliptical_prior(mean, cov)
    key, hist, subiter = _native_run("elliptical_slice", rng_key, eng, q, num_steps, thin, keep_history, chain_offset,
                                     torch.int32)
    check(lib().bjx_elliptical_slice_sample(eng.h, ptr(key), ptr(q), ptr(logl), int(num_steps), int(max_subiter),
                                            ptr(hist), int(thin), ptr(subiter)), eng.h)
    return EllipSliceState(q, logl), hist, subiter


def sample_slice_sampling_native(rng_key, state, logdensity_fn, num_steps, *, scale=1.0, width=1.0, interval=None,
                                 max_expansions=10, max_shrinkage=100, thin=1, keep_history=True, chain_offset=0,
                                 evaluations=None):
    """``run_inference_algorithm`` for slice sampling without a Python-level loop (libbjx ``bjx_slice_sample``): the
    same draws as ``num_steps`` calls of ``slice_sampling(logdensity_fn, proposal_generator=direction_proposal(scale),
    width=width, interval=interval, ...)`` with the step keys ``split(rng_key, T)[t]``.  ``interval`` is ``doubling``
    (the default) or ``stepping_out`` of :mod:`blackjax_b200.mcmc.slice`; ``width`` a scalar or [C].  ``evaluations``
    (optional) is a uint64 [1] CUDA tensor to which the call adds the target evaluations it made.  Returns (final
    SliceState, positions [num_steps // thin, C, D] or None, num_expansions int32 [num_steps, C], num_shrink int32
    [num_steps, C])."""
    from ._engine import get_engine
    from ._lib import check, lib, ptr
    from .mcmc.slice import SliceState, _check_caps, _interval_code
    code = _interval_code(interval)
    _check_caps(max_expansions, max_shrinkage)
    q, logp = (t.clone() for t in state)
    eng = get_engine(q, logdensity_fn)
    eng.ensure_slice_scale(scale)
    key, hist, n_exp, n_shrink = _native_run("slice_sampling", rng_key, eng, q, num_steps, thin, keep_history,
                                             chain_offset, torch.int32, torch.int32)
    w, w_dev = eng._eps(width, "width")
    check(lib().bjx_slice_sample(eng.h, ptr(key), ptr(q), ptr(logp), int(num_steps), w, ptr(w_dev), code,
                                 int(max_expansions), int(max_shrinkage), ptr(hist), int(thin), ptr(n_exp),
                                 ptr(n_shrink), ptr(evaluations)), eng.h)
    eng._width_keepalive = w_dev  # the launches are asynchronous
    return SliceState(q, logp), hist, n_exp, n_shrink


def sample_random_walk_native(rng_key, state, logdensity_fn, num_steps, *, proposal, proposal_logdensity_fn=None,
                              thin=1, keep_history=True, chain_offset=0):
    """``run_inference_algorithm`` for random-walk Metropolis without a Python-level loop (libbjx ``bjx_rw_sample``):
    the same draws as ``num_steps`` step calls with the step keys ``split(rng_key, T)[t]``.  ``proposal`` is a
    descriptor of :mod:`blackjax_b200.mcmc.random_walk` (``normal``, ``gaussian_proposal`` or
    ``gaussian_distribution``) and ``proposal_logdensity_fn`` None or its ``gaussian_logdensity``.  Returns (final
    RWState, positions [num_steps // thin, C, D] or None, acceptance rates [num_steps, C])."""
    from ._engine import get_engine
    from ._lib import check, lib, ptr
    from .mcmc.random_walk import RWState, _correct_of, _proposal_of
    kind, sigma, mean = _proposal_of(proposal, getattr(proposal, "rw_role", "proposal"))
    correct = _correct_of((kind, sigma, mean), proposal_logdensity_fn)
    q, logp = (t.clone() for t in state)
    eng = get_engine(q, logdensity_fn)
    eng.ensure_rw_proposal(kind, sigma, mean)
    key, hist, acc = _native_run("random_walk", rng_key, eng, q, num_steps, thin, keep_history, chain_offset,
                                 torch.float32)
    check(lib().bjx_rw_sample(eng.h, ptr(key), ptr(q), ptr(logp), int(num_steps), int(correct), ptr(hist), int(thin),
                              ptr(acc)), eng.h)
    return RWState(q, logp), hist, acc


def run_inference_algorithm(rng_key, inference_algorithm, num_steps, initial_state=None, initial_position=None,
                            transform=lambda state, info: (state, info), collect=True):
    """``keys = split(rng_key, num_steps)`` then ``num_steps`` calls of ``step`` (util.py:200-211).
    Each step key is split into one key per chain (step-major schedule).  ``transform`` picks what is kept;
    with ``collect=False`` only the final state is returned."""
    if (initial_state is None) == (initial_position is None):
        raise ValueError("Either `initial_state` or `initial_position` must be specified, but not both.")
    if initial_state is None:
        initial_state = inference_algorithm.init(initial_position)
    keys = bjx_random.split(rng_key, num_steps)
    state = initial_state
    history = []
    for t in range(num_steps):
        state, info = inference_algorithm.step(keys[t], state)
        if collect:
            history.append(transform(state, info))
    return state, history
