"""CPU tests of the LAPS restatement (oracle/laps.py): the reference's #969 known answer, the history and
its contraction, the bisection, the early-stop index, the key layout and rademacher."""
import numpy as np

from oracle import laps as ol
from oracle import prng as oprng
from oracle import targets as otargets

F = np.float32


def test_nan_fix_969_halves_the_step_size():
    """tests/mcmc/test_mclmc_nan_fix_969.py:253-295: at eps = 100 on the bounded target some chains report NaN, keep their
    state and the update halves the step size."""
    N, D = 16, 2
    tgt = otargets.BoundedGaussian(D)
    q = (0.5 * np.random.default_rng(0).standard_normal((N, D))).astype(F)
    state, _ = ol.initialize(q, tgt)
    ad = ol.BurnIn(D, 2)
    ad.eps = F(100.0)
    new, info = ol.burn_in_kernel(ol.sampling_keys(oprng.key(3), N, 10, 0), state, tgt, ad.L, ad.eps)
    Et = ol.summaries(new, info)
    assert Et["nans"] > 0
    bad = ~info.nonans
    np.testing.assert_array_equal(new[1][bad], state[1][bad])  # the momentum is kept too
    ol.update(ad, Et, 1.9, 0.1, 3)
    assert ad.eps == F(50.0)


def test_history_and_contraction_against_direct_numpy():
    rs = np.random.default_rng(1)
    hist, w = np.zeros((4, 3), F), np.zeros(4, F)
    rows = []
    for t in range(6):
        x = rs.standard_normal(3).astype(F)
        rows.insert(0, x)
        hist, w = ol.update_history(x, hist), ol.update_history(F(1), w)
        kept = np.array(rows[:4], np.float64)
        np.testing.assert_array_equal(hist[:len(kept)], kept.astype(F))
        a, a2 = kept.mean(0), (kept ** 2).mean(0)
        r = (a2 - a * a) / (a * a)
        np.testing.assert_allclose(ol.contract_history(hist, w), [r.max(), r.mean()], rtol=1e-12)


def test_bisection_hand_checked():
    upd = ol.bisection(0.7)
    st = ((-np.inf, np.inf), False)
    st, e = upd(st, 1.0, 0.9)        # too high: lower = 0, eps = exp(log 2)
    assert st[0] == (0.0, np.inf) and np.isclose(e, 2.0)
    st, e = upd(st, e, 0.2)          # too low: upper = log 2, bracketed: eps = exp(log 2 / 2)
    assert np.isclose(e, np.sqrt(2.0)) and not st[1]
    st, e2 = upd(st, e, 0.71)        # within 0.03: terminated, but this step still bisects (old flag)
    assert st[1] and np.isclose(e2, 2 ** 0.75)
    st, e3 = upd(st, e2, 0.1)
    assert e3 == e2


def test_stop_index():
    r = [0.5, 0.2, 0.005, 0.001, 0.5]
    assert ol.stop_index(r, 2, 0.01, 5) == 3
    assert ol.stop_index(r, 4, 0.01, 5) == 5                 # r_max > r_end at t = 4
    assert ol.stop_index([0.5, np.nan, 0.5], 1, 0.01, 3) == 2  # NaN > r_end is false: stop
    assert ol.stop_index([0.001, 0.5], 0, 0.01, 2) == 0        # save_num = 0: the probe of step 0 decides
    assert ol.stop_index([0.5, 0.5, 0.5], 1, 0.01, 3) == 3


def test_split_shape_is_the_flat_split():
    k = oprng.key(7)
    N, T = 5, 4
    flat = oprng.split(k, N * T).reshape(N, T, 2)
    for t in range(T):
        np.testing.assert_array_equal(oprng.fold_in(k, np.arange(N) * T + t), flat[:, t])
        np.testing.assert_array_equal(ol.sampling_keys(k, N, T, t),
                                      oprng.split(oprng.split(k, 2)[0], N * T).reshape(N, T, 2)[:, t])


def test_rademacher_is_two_bernoulli_minus_one():
    key = oprng.key(11)
    z = ol.rademacher(key, (100, 7))
    b = oprng.uniform(key, (100, 7)) < F(0.5)
    np.testing.assert_array_equal(z, 2 * b.astype(F) - 1)
    assert set(np.unique(z)) == {-1.0, 1.0}
