"""CPU tests of the diagonal-metric ChEES restatement (oracle/chees.py) against float64 numpy, its identity-metric limits,
and the argument checks of chees_adaptation."""
import numpy as np
import pytest

from oracle import adaptation as oadapt
from oracle import chees as ochees
from oracle import prng as oprng
from oracle import targets as otargets

F = np.float32


def test_welford_fold_matches_float64_variance():
    x = (np.random.default_rng(0).standard_normal((3000, 7)) * np.logspace(-1, 1, 7) + 3.0).astype(F)
    w = oadapt.welford_init(7)
    for chunk in np.split(x, 3):
        w = ochees.welford_fold(w, chunk)
    assert w.n == 3000
    np.testing.assert_allclose(w.m2 / (w.n - 1), np.var(x.astype(np.float64), axis=0, ddof=1), rtol=1e-5)
    np.testing.assert_allclose(w.mean, x.astype(np.float64).mean(0), rtol=1e-5, atol=1e-6)


def test_cgl_update_batch_matches_np_cov():
    rng = np.random.default_rng(1)
    D = 9
    A = rng.standard_normal((D, D))
    x = (rng.standard_normal((2500, D)) @ A.T + 5.0).astype(F)
    b = oadapt.moment_block_init(D)
    for chunk in np.array_split(x, 4):
        b = oadapt.cgl_update_batch(b, chunk)
    ref = np.cov(x.astype(np.float64), rowvar=False)
    assert b.count == 2500
    assert np.max(np.abs(b.m2 / (b.count - 1) - ref)) <= 1e-5 * np.max(np.diag(ref))


def test_power_iteration_matches_eigvalsh_with_spectral_gap():
    rng = np.random.default_rng(2)
    D = 40
    Q, _ = np.linalg.qr(rng.standard_normal((D, D)))
    ev = np.concatenate([[20.0], np.linspace(0.5, 2.0, D - 1)])
    M = ((Q * ev) @ Q.T).astype(F)
    lam, v = ochees.power_iteration(M, ochees.eig_state_init(D).eigenvector, 20)
    top = np.linalg.eigvalsh(M.astype(np.float64))[-1]
    assert abs(lam - top) <= 1e-4 * top
    assert abs(abs(float(np.dot(v, Q[:, 0]))) - 1.0) < 1e-4
    # a zero matrix: the norm guard keeps v finite and lambda floors at 1e-6
    e = ochees.recompute_eig(oadapt.moment_block_init(3), np.ones(3, F), ochees.eig_state_init(3))
    assert e.lambda_max == F(1e-6) and np.all(np.isfinite(e.eigenvector))


@pytest.mark.parametrize("T,lam,engaged,enable,max_lf,eps,consumed,clipped", [
    (1.0, 4.0, True, True, 1000, 0.1, np.pi, False),        # floor binds
    (5.0, 4.0, True, True, 1000, 0.1, 5.0, False),          # adapted length above the floor
    (1.0, 4.0, False, True, 1000, 0.1, 1.0, False),         # not engaged: no floor
    (1.0, 4.0, True, False, 1000, 0.1, 1.0, False),         # floor disabled: unchanged
    (1.0, 400.0, True, True, 100, 0.2, 20.0, True),         # floor (31.4) above the cap (20): clipped by the cap
    (30.0, 400.0, False, True, 100, 0.2, 20.0, False),      # the cap applies whenever the floor is enabled
])
def test_length_floor_truth_table(T, lam, engaged, enable, max_lf, eps, consumed, clipped):
    c, k = ochees.apply_length_floor(F(T), F(lam), engaged, enable, max_lf, F(eps))
    assert abs(float(c) - consumed) <= 1e-6 * consumed and k == clipped


@pytest.mark.parametrize("D,thresh", [(1, 64), (100, 64), (1024, 64), (1025, 64), (1089, 66), (10000, 200)])
def test_engagement_threshold(D, thresh):
    assert ochees.engagement_threshold(D) == thresh


def test_engaged_metric_and_fallback():
    w = ochees.welford_fold(oadapt.welford_init(3), np.random.default_rng(3).standard_normal((63, 3)).astype(F))
    assert np.array_equal(ochees.diagonal_imm(w, 64, 3), np.ones(3, F))
    w = ochees.welford_fold(w, np.zeros((1, 3), F))
    np.testing.assert_array_equal(ochees.diagonal_imm(w, 64, 3), np.maximum(w.m2 / F(63), F(1e-20)))


def _update_inputs(C=300, D=6, seed=4):
    rng = np.random.default_rng(seed)
    q = rng.standard_normal((C, D)).astype(F)
    return dict(prop_q=(q + rng.standard_normal((C, D)) * 0.3).astype(F), prop_p=rng.standard_normal((C, D)).astype(F),
                init_q=q, acc=rng.uniform(0.2, 1.0, C).astype(F), is_div=rng.uniform(size=C) < 0.05)


def test_whitened_criterion_with_ones_is_bit_identical_to_raw():
    s = ochees.chees_init(0.1)
    a = _update_inputs()
    for _ in range(5):
        raw = ochees.chees_update(s, **a, lr=0.1)
        w = ochees.chees_update(s, **a, imm=np.ones(6, F), whiten=True, lr=0.1)
        u = ochees.chees_update(s, **a, imm=np.full(6, 4.0, F), whiten=False, lr=0.1)
        for x, y, z in zip(raw, w, u):
            assert np.array_equal(np.asarray(x), np.asarray(y)) and np.array_equal(np.asarray(x), np.asarray(z))
        s = raw
    # a non-trivial metric changes the criterion (|dx|^2 terms measured in the metric's geometry): Adam's first moment
    v = ochees.chees_update(ochees.chees_init(0.1), **a, imm=np.logspace(-1, 1, 6).astype(F), lr=0.1)
    assert v.optim.mu != ochees.chees_update(ochees.chees_init(0.1), **a, lr=0.1).optim.mu


def test_window_fraction_one_is_bit_identical_to_none():
    tgt = otargets.DiagGaussian(np.array([0.5, 1.0, 3.0]))
    q = np.random.default_rng(5).standard_normal((64, 3)).astype(F)
    kw = dict(lr=0.2, num_steps=40)
    tr0, tr1 = [], []
    st0, eps0, nlf0, s0 = ochees.chees_run(tgt, oprng.key(3), q, 0.1, trace=tr0, **kw)
    r1 = ochees.chees_run(tgt, oprng.key(3), q, 0.1, mass_matrix_estimation="diagonal", window_fraction=1.0, trace=tr1, **kw)
    assert np.array_equal(st0.position, r1.state.position) and eps0 == r1.step_size
    assert all(a[1] == b[1] and all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(a[0], b[0]))
               for a, b in zip(tr0, tr1))
    assert np.array_equal(r1.inverse_mass_matrix, np.ones(3, F)) and not any(t[3] for t in tr1)
    # the final count goes through the floor's min/max and exp(T_ma) / exp(eps_ma) (:979-991): equal to rounding
    assert abs(r1.num_leapfrog_steps / nlf0 - 1) < 1e-5 and not r1.floor_clipped_by_cap


def test_oracle_metric_run_engages_and_floors():
    D = 4
    tgt = otargets.DiagGaussian(np.array([0.1, 1.0, 3.0, 10.0]))
    q = (np.random.default_rng(6).standard_normal((128, D)) * np.array([0.1, 1.0, 3.0, 10.0])).astype(F)
    tr = []
    r = ochees.chees_run(tgt, oprng.key(4), q, 0.05, lr=0.2, num_steps=80, mass_matrix_estimation="diagonal", trace=tr)
    assert not tr[38][3] and tr[40][3]                     # window from step 40; 128 chains >= 64 after one fold
    assert tr[64][2] != 1.0 and tr[63][2] == 1.0           # the first recompute is at step 64
    np.testing.assert_allclose(r.inverse_mass_matrix, np.array([0.1, 1.0, 3.0, 10.0]) ** 2, rtol=0.3)
    assert np.isfinite(r.num_leapfrog_steps) and r.lambda_max > 0


@pytest.mark.parametrize("kw,msg", [(dict(mass_matrix_estimation="dense"), "mass_matrix_estimation"),
                                    (dict(mass_matrix_estimation="diagonal", mass_matrix_window_fraction=1.5), "fraction"),
                                    (dict(mass_matrix_estimation="diagonal", mass_matrix_window_fraction=-0.1), "fraction")])
def test_chees_adaptation_argument_errors(kw, msg):
    import blackjax_b200 as bj
    with pytest.raises(ValueError, match=msg):
        bj.chees_adaptation(bj.targets.DiagGaussian(np.ones(2)), 8, **kw)
    with pytest.raises(ValueError, match=msg):
        ochees.chees_run(None, oprng.key(0), np.zeros((2, 2), F), 0.1, lr=0.1, num_steps=1,
                         **{("window_fraction" if k == "mass_matrix_window_fraction" else k): v for k, v in kw.items()})
