"""CPU tests of the adjusted MCLMC tuner's restatement (oracle/adjusted_mclmc_tuning.py): stage lengths,
the masked dual averaging with its clamp and log round trip, the L / step-size update order, the key tree against an explicit
oprng composition, handle_nans' revert, the exit invariant, the reference's L / step = 2.0 and 1.5 assertions at D = 5, and
the Python surface of blackjax_b200.adjusted_mclmc_find_L_and_step_size without a GPU, and a spill-free sm_90a compile of
every instance of the fused tuning step beside the transition it shares its body with."""
import inspect
import os

import numpy as np
import pytest

from oracle import adjusted_mclmc as ao
from oracle import adjusted_mclmc_tuning as at
from oracle import prng as oprng
from oracle import targets as otargets
from oracle.adaptation import DAState, da_init, da_update
from test_kernel_spills import (AMCLMC_TRANSITION, INSTANCES, NVCC, WITH_CSRC, assert_entries_clean, instantiate,
                                ptxas_log)

F = np.float32
MCLACHLAN = (0.1931833275037836, 0.5, 1.0 - 2 * 0.1931833275037836, 0.5, 0.1931833275037836)
UNIFORM0 = ("uniform", 0)  # the reference tests' ceil(uniform(key) * rescale(avg)), unclipped


def _dyn_state(C, D, seed, scale=1.0):
    rs = np.random.default_rng(seed)
    tgt = otargets.DiagGaussian(np.full(D, scale))
    q = rs.standard_normal((C, D)).astype(F)
    logp, g = tgt(q)
    return tgt, (q, logp, g, oprng.split(oprng.key(seed + 100), C))


def test_stage_lengths_truncate_after_dividing_by_the_windows():
    assert at.stage_lengths(4000, 0.1, 0.1, 0.0) == (400, 400, 0)
    assert at.stage_lengths(999, 0.1, 0.1, 0.1) == (99, 99, 99)  # int(), not round(): 99.9 -> 99
    assert at.stage_lengths(1000, 0.1, 0.2, 0.1, num_windows=3) == (33, 66, 33)
    assert at.stage_lengths(25, 0.1, 0.1, 0.0) == (2, 2, 0)
    from blackjax_b200.adaptation import adjusted_mclmc_adaptation as ama
    for args in ((4000, 0.1, 0.1, 0.0), (999, 0.1, 0.1, 0.1), (1000, 0.1, 0.2, 0.1, 3), (7, 0.3, 0.0, 0.5, 2)):
        assert ama.stage_lengths(*args) == at.stage_lengths(*args)


def test_masked_dual_averaging_clamp_and_log_round_trip():
    C = 4
    eps = np.array([0.1, 0.5, 1.0, 2.0], F)
    da = tuple(np.broadcast_to(np.asarray(x, F), (C,)).copy() for x in da_init(eps))
    acc = np.array([0.1, 0.9, 0.5, 0.0], F)
    new = at.da_update_masked(da, acc, 0.65, np.array([1, 0, 1, 0], bool))
    ref = DAState(*da_update(DAState(*da), acc, target=0.65))
    for f, r, o in zip(new, ref, da):
        np.testing.assert_array_equal(f[[0, 2]], np.asarray(r, F)[[0, 2]])
        np.testing.assert_array_equal(f[[1, 3]], o[[1, 3]])
    # clamp(1e-5, exp(log_step), L / 1.1) with the float32 1.1, then log: the round trip may move log_step by an ulp
    L = np.array([1.0, 1.0, 1e-3, 1.0], F)
    step, log_step = at.clamp_step(np.array([np.log(0.3), 5.0, 0.0, -40.0], F), L)
    np.testing.assert_array_equal(step, np.array([np.exp(F(np.log(0.3))), F(1.0) / F(1.1), F(1e-3) / F(1.1), F(1e-5)], F))
    np.testing.assert_array_equal(log_step, np.log(step))


def test_fix_L_false_updates_L_with_the_old_step_size():
    """test_inner_fn_fix_L_false_updates_L restated: with fix_L = False L moves as step / old step, the old step taken
    before the update (the reference's ordering fix, :20-23, :294-299); with fix_L = True it stays."""
    C, D = 3, 5
    tgt, st = _dyn_state(C, D, 1)
    keys = oprng.split(oprng.key(2), C)
    eps, L = np.full(C, 0.1, F), np.full(C, 1.0, F)
    da = tuple(np.broadcast_to(np.asarray(x, F), (C,)).copy() for x in da_init(eps))
    streaming = (np.zeros(C, F), np.zeros((C, 2, D), F))
    out = at.tune_step(UNIFORM0, keys, st, tgt, F(1), eps, L, da, streaming, 1.0, False, 0.65, MCLACHLAN)
    _, e2, L2 = out[:3]
    np.testing.assert_array_equal(L2, (L * (e2 / eps).astype(F)).astype(F))
    assert not np.allclose(L2, L, rtol=1e-3)
    out = at.tune_step(UNIFORM0, keys, st, tgt, F(1), eps, L, da, streaming, 1.0, True, 0.65, MCLACHLAN)
    np.testing.assert_array_equal(out[2], L)
    # a masked-out step (m = 0) keeps eps and L, and the DA state, except the log round trip of log_step
    out = at.tune_step(UNIFORM0, keys, st, tgt, F(1), eps, L, da, streaming, 0.0, False, 0.65, MCLACHLAN)
    np.testing.assert_array_equal(out[1], eps)
    np.testing.assert_array_equal(out[2], L)
    for a, b in zip(out[3][1:], da[1:]):
        np.testing.assert_array_equal(a, b)
    # and accumulates (x, x^2) with weight success * step
    _, step = None, at.clamp_step(da[0], L)[0]
    np.testing.assert_array_equal(out[4][0], step)


def test_inner_adaptation_moves_L_over_a_pass():
    """The reference's own regression (fix_L_first_da = False, frac_tune2 = 0, L = 1, step = 0.1, 800 steps) on a pass."""
    C, D = 2, 5
    tgt, st = _dyn_state(C, D, 3)
    base = oprng.split(oprng.key(4), C)
    _, _, L, _, _ = at._pass(UNIFORM0, base, 800, 800, st, tgt, F(1), np.full(C, 0.1, F), np.full(C, 1.0, F), False,
                             0.65, MCLACHLAN, np.zeros(C, F))
    assert not np.allclose(L, 1.0, rtol=1e-3)


def test_key_tree_against_explicit_oprng_composition():
    """Pass-1 step t of window i uses split(p1, n1 + n2)[t] with p1, p2 = split(split(fold_in(part1, i))[1]); stage 3
    transitions use split(k1, n3)[t] with k1, k2 = split(fold_in(part2, i)); split(key, n)[i] = fold_in(key, i)."""
    k = oprng.split(oprng.key(9), 3)
    part1, part2 = oprng.split(k, 2)[:, 0], oprng.split(k, 2)[:, 1]
    for i in range(3):
        wk = oprng.fold_in(part1, i)
        check_rk = oprng.split(wk, 2)
        p = oprng.split(check_rk[:, 1], 2)
        for n, t in ((10, 0), (10, 7)):
            want = oprng.split(p[:, 0], n)[:, t]
            np.testing.assert_array_equal(oprng.fold_in(p[:, 0], t), want)
        np.testing.assert_array_equal(oprng.fold_in(oprng.fold_in(wk, 1), 0), p[:, 0])
        np.testing.assert_array_equal(oprng.fold_in(oprng.fold_in(wk, 1), 1), p[:, 1])
    # the stage-3 window key of the adaptation that follows is k2 = split(part2)[1] = fold_in(part2, 1)
    np.testing.assert_array_equal(oprng.split(part2, 2)[:, 1], oprng.fold_in(part2, 1))


class _NaNBeyond:
    """A Gaussian whose position goes non-finite beyond |x| > 3 (the proposal is then inf)."""

    def __call__(self, q):
        q = np.asarray(q, F)
        bad = np.any(np.abs(q) > 3, axis=1)
        logp = np.where(bad, F(np.inf), (-0.5 * (q * q).sum(1)).astype(F)).astype(F)
        g = np.where(bad[:, None], F(np.inf), -q).astype(F)
        return logp, g


def test_handle_nans_reverts_the_whole_state_including_the_key():
    C, D = 4, 3
    q = np.zeros((C, D), F)
    prev = (q, np.zeros(C, F), np.zeros((C, D), F), oprng.split(oprng.key(1), C))
    new = (np.where(np.arange(C)[:, None] % 2 == 0, F(np.inf), F(1.0)).astype(F) * np.ones((C, D), F),
           np.full(C, F(np.nan)), np.full((C, D), F(np.nan)), oprng.split(oprng.key(2), C))
    nonans, st = at.handle_nans(prev, new)
    np.testing.assert_array_equal(nonans, [False, True, False, True])
    for a, b in zip(st, prev):
        np.testing.assert_array_equal(a[~nonans], b[~nonans])
    np.testing.assert_array_equal(st[3][nonans], new[3][nonans])
    assert np.all(st[1][nonans] == 0) and np.all(st[2][nonans] == 0)


def test_exit_invariant_and_the_reference_ratios_at_dim_5():
    """test_tuner_returns_L_over_step_approx_target / _target_1p5 / _default_is_target_2 (:144-195) on 3 chains each."""
    C, D = 3, 5
    for tk, seed in ((2.0, 11), (1.5, 12)):
        tgt, st = _dyn_state(C, D, seed)
        keys = oprng.split(oprng.key(seed), C)
        _, (L, eps, imm), count = at.find_L_and_step_size(UNIFORM0, keys, 4000, st, tgt, MCLACHLAN, 0.65,
                                                          target_num_integration_steps=tk)
        np.testing.assert_allclose(L / eps, tk, rtol=1e-5)
        np.testing.assert_array_equal(L, (F(tk) * eps).astype(F))
        assert np.all(eps > 0.1) and np.all(np.isfinite(imm)) and np.all(count > 0)


def test_static_kernel_reports_the_float_avg():
    C, D = 3, 4
    tgt, st = _dyn_state(C, D, 5)
    avg = np.array([2.0, 2.0000002, 1.9999999], F)
    n, rep = at.num_steps_of(("static", None), avg, None)
    np.testing.assert_array_equal(n, [2, 3, 2])
    np.testing.assert_array_equal(rep, avg)
    _, (L, eps, _), count = at.find_L_and_step_size(("static", None), oprng.split(oprng.key(5), C), 200, st[:3], tgt,
                                                    MCLACHLAN, 0.9, frac_tune3=0.1)
    np.testing.assert_allclose(L / eps, 2.0, rtol=1e-6)
    assert count.dtype == F and np.all(count > 0)


def test_public_signature_and_rejections_without_gpu():
    import blackjax_b200 as bj
    from blackjax_b200.adaptation import adjusted_mclmc_adaptation as ama
    params = list(inspect.signature(bj.adjusted_mclmc_find_L_and_step_size).parameters.values())
    names = [p.name for p in params]
    assert names[:15] == ["mclmc_kernel", "logdensity_fn", "num_steps", "state", "rng_key", "target", "frac_tune1",
                          "frac_tune2", "frac_tune3", "diagonal_preconditioning", "params", "max", "num_windows",
                          "tuning_factor", "target_num_integration_steps"]
    defaults = {p.name: p.default for p in params}
    assert (defaults["frac_tune1"], defaults["frac_tune2"], defaults["frac_tune3"], defaults["max"],
            defaults["num_windows"], defaults["tuning_factor"], defaults["target_num_integration_steps"]) == (
        0.1, 0.1, 0.0, "avg", 1, 1.3, 2.0)
    assert params[-1].kind == inspect.Parameter.KEYWORD_ONLY and params[-1].name == "max_history_bytes"
    with pytest.raises(TypeError):
        ama._kernel_rule(bj.hmc.build_kernel())
    with pytest.raises(ValueError):
        ama._kernel_rule(bj.adjusted_mclmc_dynamic.build_kernel(integration_steps_fn=lambda k, avg: 3))
    assert ama._kernel_rule(bj.adjusted_mclmc.build_kernel()) == (False, 0, 0)
    fn = bj.mcmc.adjusted_mclmc_dynamic.make_random_trajectory_length_fn(True, min_steps=0)
    assert ama._kernel_rule(bj.adjusted_mclmc_dynamic.build_kernel(integration_steps_fn=fn)) == (True, 2, 0)
    assert ama._kernel_rule(bj.adjusted_mclmc_dynamic.build_kernel()) == (True, 1, 0)


def test_rescale_matches_the_sampler_restatement():
    for mu in (1.1, 1.5, 2.0, 2.5, 3.7, 8.0):
        assert at.num_steps_of(("uniform", 0), np.array([mu], F), oprng.split(oprng.key(1), 1))[0][0] == \
            ao.steps_uniform(oprng.split(oprng.key(1), 1), mu, 0)[0]


@pytest.mark.skipif(not os.path.exists(NVCC), reason="needs nvcc")
def test_tuning_step_compiles_without_spills(tmp_path):
    src = instantiate(("k_amclmc_tune", "Params, const uint32_t*, float*, float*, float*, AmclmcTuneArgs"),
                      AMCLMC_TRANSITION)
    log = ptxas_log(tmp_path, src, WITH_CSRC)
    assert_entries_clean(log, ("k_amclmc_tune", "k_amclmc_transition"), 4 * len(INSTANCES))
