"""CPU tests of the MCLMC tuner restatement (oracle/mclmc_tuning.py): the stage arithmetic, the clip, the
streaming-moment rules and the failure path of one tuning step, the reference's own tuner tests
(tests/mcmc/test_mclmc_nan_fix_969.py:127-176, tests/mcmc/test_sampling.py:482-557) restated on it, and the Python
surface's argument checks."""
import numpy as np
import pytest

from oracle import mclmc as om
from oracle import mclmc_tuning as ot
from oracle import prng as oprng
from oracle import targets as otargets

F = np.float32
_L = 0.1931833275037836
TABLES = {"velocity_verlet": (0.5, 1.0, 0.5), "mclachlan": (_L, 0.5, 1.0 - 2 * _L, 0.5, _L)}


def test_stage_lengths():
    from blackjax_b200.adaptation.mclmc_adaptation import stage_lengths
    cases = [  # (num_steps, f1, f2, f3, diag) -> (n1, n2, readjust, n3, count)
        ((25, 0.1, 0.1, 0.1, True), (2, 2, 1, 2, 6)),        # 2.5 rounds to 2; round(2/3) = 1 runs, 2 // 3 = 0 counts
        ((35, 0.1, 0.1, 0.1, True), (4, 4, 1, 4, 13)),       # 3.5 rounds to 4
        ((1000, 0.1, 0.1, 0.1, True), (100, 100, 33, 100, 333)),
        ((1000, 0.1, 0.1, 0.1, False), (100, 100, 0, 100, 300)),
        ((10, 0.1, 0.1, 0.1, True), (1, 1, 0, 1, 2)),        # n2 <= 1: no readjustment; n3 < 2: no stage 3
        ((60, 1.0, 0.0, 0.0, False), (60, 0, 0, 0, 60)),
        ((50, 0.1, 0.1, 0.03, True), (5, 5, 2, 2, 13)),      # 1.5 rounds to 2; round(5/3) = 2 runs, 5 // 3 = 1 counts
    ]
    for args, want in cases:
        assert stage_lengths(*args) == want, args
        assert ot.stage_lengths(*args) == want, args


def test_clip_rule():
    inf = F(np.inf)
    np.testing.assert_array_equal(ot.clip_step_size([0.5, 2.0, 1.0, np.nan, 3.0], [1.0, 1.0, 1.0, 1.0, inf]),
                                  np.array([0.5, 1.0, 0.0, 0.0, 3.0], F))
    assert ot.clip_step_size(inf, inf) == 0  # equal: neither predicate holds


def test_safediv_zero_and_the_weight_zero_update():
    assert ot.safediv(F(0), F(0)) == 0 and ot.safediv(F(0), F(3)) == 0
    total, m = ot.incremental_value_update(np.zeros((1, 3), F), np.zeros(1, F), np.zeros((1, 2, 3), F), np.zeros(1, F))
    assert total[0] == 0 and np.all(m == 0)
    # total > 0, weight 0: (total av) / total is evaluated and need not return av exactly
    av = np.array([[[0.1, 0.7, 1.3], [0.2, 0.3, 0.4]]], F)
    tot = np.array([F(3.3)], F)
    _, m = ot.incremental_value_update(np.ones((1, 3), F), tot, av, np.zeros(1, F))
    np.testing.assert_array_equal(m, ((tot[0] * av).astype(F) / tot[0]).astype(F))


def _gauss_state(C, D, seed=0):
    target = otargets.StdNormal(D)
    keys = oprng.split(oprng.key(seed), C)
    q = np.random.default_rng(seed).standard_normal((C, D)).astype(F)
    return target, om.mclmc_init(q, target, keys)


def test_first_step_and_weight_use_the_new_step_size():
    C, D = 4, 6
    target, state = _gauss_state(C, D)
    k = ot.Constants(D)
    adaptive = (np.zeros(C, F), np.zeros(C, F), np.full(C, np.inf, F))
    streaming = (np.zeros(C, F), np.zeros((C, 2, D), F))
    keys = oprng.split(oprng.key(7), C)
    new_state, eps, adaptive, (total, m), ok = ot.tune_step(keys, state, target, np.ones(D, F), F(2.0), F(0.5),
                                                            adaptive, streaming, 1.0, TABLES["mclachlan"], np.inf, k)
    assert np.all(ok) and np.all(np.isfinite(eps)) and np.all(eps > 0)  # eps_max = inf does not poison the first step
    np.testing.assert_array_equal(total, eps)  # weight = mask * success * (new step size)
    np.testing.assert_allclose(m[:, 0], new_state[0], rtol=1e-6)
    np.testing.assert_allclose(m[:, 1], new_state[0] ** 2, rtol=1e-6)


def test_failed_step_restores_the_previous_momentum():
    """#969 (test_mclmc_nan_fix_969.py:127-160): step size 100 on the bounded target diverges; the tuner keeps the whole
    previous state, momentum included, and step_size_max becomes 0.8 * 100."""
    target = otargets.BoundedGaussian(2)
    init_key, step_key, _ = oprng.split(oprng.key(0), 3)
    state = om.mclmc_init(np.zeros((1, 2), F), target, init_key[None])
    _, info = om.mclmc_kernel(step_key[None], state, target, np.ones(2, F), F(1.0), F(100.0), TABLES["mclachlan"])
    assert not info.nonans[0]
    k = ot.Constants(2)
    # whichever key diverges, a failed step keeps the state; find one that does
    seeds = [s for s in range(20)
             if not ot.tune_step(oprng.key(s)[None], state, target, np.ones(2, F), F(1.0), F(100.0),
                                 (np.zeros(1, F), np.zeros(1, F), np.full(1, np.inf, F)),
                                 (np.zeros(1, F), np.zeros((1, 2, 2), F)), 1.0, TABLES["mclachlan"], np.inf, k)[4][0]]
    assert seeds
    new_state, eps, (time, x_avg, eps_max), (total, m), ok = ot.tune_step(
        oprng.key(seeds[0])[None], state, target, np.ones(2, F), F(1.0), F(100.0),
        (np.zeros(1, F), np.zeros(1, F), np.full(1, np.inf, F)), (np.zeros(1, F), np.zeros((1, 2, 2), F)), 1.0,
        TABLES["mclachlan"], np.inf, k)
    assert not ok[0] and eps_max[0] == F(80.0) and eps[0] <= 80.0
    for a, b in zip(new_state, state):
        np.testing.assert_array_equal(a, b)
    assert total[0] == 0 and np.all(m == 0)  # weight 0 and total 0: the safediv zero


def test_degenerate_dimension_gives_infinite_L():
    C, D = 2, 4
    target, state = _gauss_state(C, D, seed=1)
    imm = np.ones(D, F)
    imm[2] = 0  # the position never moves along dim 2: its ESS is 0
    _, (L, eps, _), _, _ = ot.find_L_and_step_size(oprng.split(oprng.key(5), C), 40, state, target, TABLES["mclachlan"],
                                                   frac_tune1=0.2, frac_tune2=0.0, frac_tune3=0.5,
                                                   diagonal_preconditioning=False, params=(F(2.0), F(0.5), imm))
    assert np.all(np.isinf(L)) and np.all(np.isfinite(eps))


def _run_969(table, seed, ss_init, num_steps=60):
    """_run_tuning of test_mclmc_nan_fix_969.py:54-74."""
    target = otargets.BoundedGaussian(2)
    init_key, tune_key = oprng.split(oprng.key(seed), 2)
    state = om.mclmc_init(np.zeros((1, 2), F), target, init_key[None])
    _, (L, eps, imm), _, _ = ot.find_L_and_step_size(tune_key[None], num_steps, state, target, TABLES[table],
                                                     frac_tune1=1.0, frac_tune2=0.0, frac_tune3=0.0,
                                                     diagonal_preconditioning=False,
                                                     params=(np.sqrt(F(2)), F(ss_init), np.ones(2, F)))
    return eps[0]


def test_adaptation_divergent_step_shrinks_step_size():
    assert _run_969("mclachlan", 0, 100.0, num_steps=3) <= 80.0


@pytest.mark.parametrize("table", ["mclachlan", "velocity_verlet"])
def test_behavioral_convergence_from_large_step_size(table):
    final = [float(_run_969(table, sd + 100, 100.0)) for sd in range(6)]
    assert all(0.1 <= s <= 10.0 for s in final), final


def test_mclmc_preconditioning():
    """test_sampling.py:482-557: D = 100, condition number 10, 20000 steps; the tuned M^-1 lines up with the eigenvalues."""
    dim, kappa = 100, 10.0
    eigs = np.logspace(-0.5 * np.log10(kappa), 0.5 * np.log10(kappa), dim).astype(F)
    target = otargets.DiagGaussian(np.sqrt(eigs.astype(np.float64)), dim)
    init_key, tune_key = oprng.split(oprng.key(2), 2)
    q0 = (oprng.normal(init_key, (dim,)) * np.max(np.sqrt(eigs))).astype(F)[None]
    state = om.mclmc_init(q0, target, init_key[None])
    _, (L, eps, imm), _, _ = ot.find_L_and_step_size(tune_key[None], 20000, state, target, TABLES["mclachlan"],
                                                     diagonal_preconditioning=True)
    m2 = imm[0].astype(np.float64) ** 2
    assert abs(np.dot(m2 / np.linalg.norm(m2), eigs / np.linalg.norm(eigs)) - 1) < 0.1


def test_python_surface_without_gpu():
    from blackjax_b200.adaptation.mclmc_adaptation import mclmc_find_L_and_step_size
    with pytest.raises(ValueError, match="logdensity_fn is required"):
        mclmc_find_L_and_step_size(lambda *a: None, 100, None, None)
    with pytest.raises(TypeError, match="build_kernel"):
        mclmc_find_L_and_step_size(lambda *a: None, 100, None, None, logdensity_fn=object())
    import blackjax_b200 as blackjax
    assert blackjax.mclmc_find_L_and_step_size is mclmc_find_L_and_step_size
    k = blackjax.mclmc.build_kernel(chain_offset=5)
    assert k.chain_offset == 5 and len(k.coefficients) == 5
