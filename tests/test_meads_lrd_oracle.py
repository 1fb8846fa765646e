"""CPU tests of the MEADS-LRD restatement (oracle/meads_lrd.py) against float64 numpy, and the argument checks
of meads_adaptation(..., low_rank_rank=k)."""
import numpy as np
import pytest

from oracle import meads_lrd as olrd

F = np.float32


def _correlated(C, D, seed):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((D, D)) / np.sqrt(D)
    return (rng.standard_normal((C, D)) @ A.T * np.exp(rng.uniform(-1, 1, D)) + 2.0).astype(F)


def test_accumulated_metric_matches_float64():
    C, D, k = 3000, 12, 4
    x = _correlated(C, D, 0)
    acc = olrd.moment_block_init(D)
    for chunk in np.array_split(x, 3):
        acc = olrd.cgl_update_batch(acc, chunk)
    sigma, U, lam = olrd.from_accumulated(acc.m2, acc.count, k)
    cov = np.cov(x.astype(np.float64), rowvar=False)
    s64 = np.sqrt(np.diag(cov))
    R = cov / np.outer(s64, s64)
    l64, V64 = np.linalg.eigh(R)
    order = np.argsort(np.abs(l64 - 1.0))[::-1][:k]
    np.testing.assert_allclose(sigma, s64, rtol=1e-5)
    np.testing.assert_allclose(lam, l64[order], atol=1e-4)
    assert np.all(np.diff(np.abs(lam - 1.0)) <= 0)
    np.testing.assert_allclose(np.abs(np.sum(U * V64[:, order], axis=0)), 1.0, atol=1e-3)


def test_selection_order_ties_take_the_later_eigh_index():
    lam_all = np.array([0.5, 0.9, 1.5, 1.1], F)                  # scores .5 .1 .5 .1 -> [2, 0, 3]
    U, lam = olrd.select_top(lam_all, np.eye(4, dtype=F), 3)
    np.testing.assert_array_equal(lam, lam_all[[2, 0, 3]])
    np.testing.assert_array_equal(U, np.eye(4, dtype=F)[:, [2, 0, 3]])


def test_floor_fallback_and_gate():
    np.testing.assert_array_equal(olrd.floor(np.array([-1.0, 0.0, 2e-6, 3.0], F)), np.array([1e-6, 1e-6, 2e-6, 3.0], F))
    assert np.isnan(olrd.floor(np.array([np.nan], F))[0])
    x = _correlated(64, 5, 1)
    x[:, 2] = 4.0                                                  # a constant column: std 0 -> 1
    sigma, U, lam = olrd.fallback(x, 3)
    s64 = x.astype(np.float64).std(0)
    np.testing.assert_allclose(sigma[[0, 1, 3, 4]], s64[[0, 1, 3, 4]], rtol=1e-6)
    assert sigma[2] == 1.0
    np.testing.assert_array_equal(U, np.eye(5, 3, dtype=F))
    np.testing.assert_array_equal(lam, np.ones(3, F))
    acc = olrd.moment_block_init(5)
    acc, on, *_ = olrd.step_metric(acc, x[:9], 3, True)          # 9 < 2 D samples
    assert not on and acc.count == 9
    acc, on, *_ = olrd.step_metric(acc, x[9:10], 3, True)        # 10 = 2 D
    assert on
    acc2, on, *_ = olrd.step_metric(acc, x, 3, False)            # outside the window: no fold, fallback
    assert not on and acc2.count == acc.count


def test_transform_matches_float64_and_reduces_to_diagonal():
    C, D, k = 50, 8, 3
    x = _correlated(C, D, 2)
    rng = np.random.default_rng(3)
    U, _ = np.linalg.qr(rng.standard_normal((D, k)))
    U = U.astype(F)
    lam = np.array([4.0, 0.25, 2.0], F)
    sigma = np.exp(rng.uniform(-1, 1, D)).astype(F)
    got = olrd.precondition(x, sigma, U, lam)
    U64 = U.astype(np.float64)
    want = (x @ (np.eye(D) + U64 @ np.diag(1 / np.sqrt(lam) - 1) @ U64.T)) / sigma
    np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-5)
    np.testing.assert_array_equal(olrd.precondition(x, sigma, U, np.ones(k, F)), (x / sigma).astype(F))


def test_fold_parameters_with_unit_lambda_match_diagonal_heuristic_step_size():
    from oracle import meads as omeads
    C, D, K = 64, 6, 4
    x = _correlated(C, D, 4)
    g = -x
    sigma, U, lam = olrd.fallback(x, 2)
    eps, scales, alpha, delta = olrd.fold_parameters(x, g, 3, K, sigma, U, lam)
    eps0, scales0, _, _ = omeads.fold_parameters(x, g, 3, K)
    np.testing.assert_array_equal(eps, eps0)
    np.testing.assert_array_equal(scales, scales0)
    assert np.all((alpha > 0) & (alpha < 1)) and np.array_equal(delta, alpha / F(2))


def test_argument_errors():
    import blackjax_b200 as bj
    from blackjax_b200 import targets as T
    from blackjax_b200.adaptation import meads_adaptation as mm
    tgt = T.StdNormal(4)
    with pytest.raises(ValueError, match="low_rank_rank"):
        bj.meads_adaptation(tgt, 1, num_folds=1, low_rank_rank=3)
    with pytest.raises(ValueError, match="low_rank_window_fraction"):
        bj.meads_adaptation(tgt, 8, num_folds=2, low_rank_rank=3, low_rank_window_fraction=-0.1)
    with pytest.raises(ValueError, match="low_rank_window_fraction"):
        bj.meads_adaptation(tgt, 8, num_folds=2, low_rank_rank=3, low_rank_window_fraction=1.5)
    bj.meads_adaptation(tgt, 8, num_folds=2, low_rank_rank=3, low_rank_window_fraction=1.0)
    with pytest.raises(NotImplementedError, match="dim <= 512"):
        mm._low_rank_limits(tgt, 3, 513)
    with pytest.raises(NotImplementedError, match="rank"):
        mm._low_rank_limits(tgt, 17, 100)
    user = T.UserTarget(4, "", dense_metric=False)
    with pytest.raises(NotImplementedError, match="dense_metric"):
        mm._low_rank_limits(user, 3, 4)
    mm._low_rank_limits(tgt, 16, 512)
