"""CPU tests of the low-rank window adaptation's oracle (oracle/low_rank_window.py) -- the reference's own
known answers (tests/adaptation/test_low_rank_adaptation.py) -- of the accumulator form the device computes, of the
package's schedule and retained-step rule, and of the argument checks."""
import numpy as np
import pytest

import blackjax_b200 as bj
from blackjax_b200.adaptation import low_rank_adaptation as lra
from oracle import low_rank_window as o


def spd(rs, n):
    A = rs.standard_normal((n, n))
    return A @ A.T + n * np.eye(n)


# ---- SPD mean ------------------------------------------------------------------------------------------------------
def test_spd_mean_symmetry_commutativity_identity_equal_and_positive():
    rs = np.random.default_rng(0)
    A, B = spd(rs, 5), spd(rs, 5)
    G = o.spd_mean(A, B)
    np.testing.assert_allclose(G, G.T, atol=1e-10)
    np.testing.assert_allclose(o.spd_mean(A, B), o.spd_mean(B, A), atol=1e-9)
    A4 = spd(rs, 4)
    G = o.spd_mean(np.eye(4), A4)
    np.testing.assert_allclose(G @ G, A4, atol=1e-9)
    np.testing.assert_allclose(o.spd_mean(A4, A4), A4, atol=1e-9)
    assert np.all(np.linalg.eigvalsh(o.spd_mean(spd(rs, 6), spd(rs, 6))) > 0)


# ---- the estimator -------------------------------------------------------------------------------------------------
def buffers(seed, B, d):
    rs = np.random.default_rng(seed)
    return rs.standard_normal((B, d)), rs.standard_normal((B, d))


def test_estimator_shapes_positive_sigma_orthonormal_u_and_masking():
    x, g = buffers(1, 60, 10)
    sigma, mu, U, lam = o.compute_low_rank_metric(x, g, 60, 4, 1.0, 2.0)
    assert sigma.shape == (10,) and mu.shape == (10,) and U.shape == (10, 4) and lam.shape == (4,)
    assert np.all(sigma > 0)
    np.testing.assert_allclose(U.T @ U, np.eye(4), atol=1e-10)
    assert np.all((lam < 0.5) | (lam > 2.0) | (lam == 1.0))


def test_estimator_mu_star_and_sigma_formulas():
    x, g = buffers(2, 200, 6)
    sigma, mu, _, _ = o.compute_low_rank_metric(x, g, 200, 2, 1.0, 2.0)
    np.testing.assert_allclose(mu, x.mean(0) + sigma ** 2 * g.mean(0), rtol=1e-12)
    np.testing.assert_allclose(sigma, np.clip((x.var(0) / np.maximum(g.var(0), 1e-10)) ** 0.25, 1e-20, 1e20), rtol=1e-12)


def test_estimator_d_less_than_2k_pads_and_partial_buffer():
    x, g = buffers(3, 30, 4)
    sigma, mu, U, lam = o.compute_low_rank_metric(x, g, 30, 4, 1.0, 2.0)
    assert U.shape == (4, 4) and sigma.shape == (4,)
    x, g = buffers(4, 100, 8)
    x[40:], g[40:] = 0.0, 0.0
    sigma, mu, U, lam = o.compute_low_rank_metric(x, g, 40, 3, 1.0, 2.0)
    ref = o.compute_low_rank_metric(x[:40], g[:40], 40, 3, 1.0, 2.0)
    np.testing.assert_allclose(sigma, ref[0], rtol=1e-12)
    np.testing.assert_allclose(o.implied_inverse_mass_matrix(sigma, U, lam), o.implied_inverse_mass_matrix(*ref[:1], *ref[2:]),
                               rtol=1e-9, atol=1e-12)
    # q = min(d, 2k) < k: zero columns and ones beyond q
    x, g = buffers(5, 50, 3)
    _, _, U, lam = o.compute_low_rank_metric(x, g, 50, 5, 1.0, 2.0)
    assert np.all(U[:, 3:] == 0.0) and np.all(lam[3:] == 1.0)


@pytest.mark.parametrize("wrap", [False, True])
@pytest.mark.parametrize("d,k,C", [(6, 2, 1), (12, 3, 3), (40, 4, 2)])
def test_accumulator_form_equals_row_form(d, k, C, wrap):
    """Chan-merged (count, mean, M2) of the retained rows, x_bar = (count / n) mean and the M2 + count d d^T scatter
    give the reference's estimator on the buffer -- also when the window outgrew the buffer (the last B steps kept, the
    sums still divided by n)."""
    rs = np.random.default_rng(d * 7 + C + wrap)
    B = 30
    steps = 47 if wrap else 21
    L = rs.standard_normal((d, d)) / np.sqrt(d)
    xs = rs.standard_normal((steps, C, d)) @ L.T + 0.3
    gs = -xs * 1.7 + 0.1 * rs.standard_normal((steps, C, d))
    core = o.ResetCore(d, k, 1e-3, 2.0, B, C)
    for t in range(steps):
        core.update(xs[t], gs[t])
    core.final()
    mx, mg = o.moments_init(d), o.moments_init(d)
    for t in range(max(0, steps - B), steps):
        mx, mg = o.moments_fold(mx, xs[t]), o.moments_fold(mg, gs[t])
    sigma, mu, U, lam = o.metric_from_moments(mx, mg, C * steps, k, 1e-3, 2.0)
    np.testing.assert_allclose(sigma, core.sigma, rtol=1e-10)
    np.testing.assert_allclose(mu, core.mu_star, rtol=1e-9, atol=1e-12)
    Mr = o.implied_inverse_mass_matrix(core.sigma, core.U, core.lam)
    np.testing.assert_allclose(o.implied_inverse_mass_matrix(sigma, U, lam), Mr, rtol=1e-7, atol=1e-9 * np.abs(Mr).max())


# ---- schedules -----------------------------------------------------------------------------------------------------
def test_growing_schedule_golden_sequences_and_is_late():
    s = o.build_growing_window_schedule(5000)
    assert len(s) == 5000
    assert o.window_sizes(s) == [10] * 150 + [80, 120, 180, 270, 405, 608, 1087]
    assert sum(1 for st, _ in s if st == 0) == 750
    for n, last in {1000: 350, 2000: 450, 5000: 1087}.items():
        assert o.window_sizes(o.build_growing_window_schedule(n))[-1] == last
    s = o.build_growing_window_schedule(2000)
    assert all(st == 0 and not e for st, e in s[2000 - 300:])
    assert s[0][0] == 1 and bj.build_schedule(1000)[0][0] == 0
    for n in (1, 5, 19, 20, 21):
        assert len(o.build_growing_window_schedule(n)) == n


@pytest.mark.parametrize("n", [1, 5, 19, 20, 21, 50, 120, 200, 1000, 2000, 5000])
@pytest.mark.parametrize("kw", [{}, {"early_window": 0.5, "step_size_window": 0.2}, {"window_growth": 2.0, "window_size": 7}])
def test_package_growing_schedule_matches_oracle(n, kw):
    assert [(int(a), bool(b)) for a, b in bj.build_growing_window_schedule(n, **kw)] == o.build_growing_window_schedule(n, **kw)


@pytest.mark.parametrize("n", [20, 120, 1000, 3000])
@pytest.mark.parametrize("growing", [False, True])
def test_retained_steps_are_what_the_buffer_holds_at_each_window_end(n, growing):
    sched = bj.build_growing_window_schedule(n) if growing else bj.build_schedule(n)
    b = lra.schedule_bytes(sched, n)
    B = o.buffer_size(n)
    assert lra.buffer_size(n) == B
    start = None
    for t, (st, e) in enumerate(sched):
        assert b[t] & 3 == st | (int(e) << 1)
        if st == 1 and start is None:
            start = t
        if e:
            for u in range(start, t + 1):
                assert bool(b[u] & 4) == (u >= t + 1 - B)
            start = None
    if n == 1000 and not growing:   # the last Stan window (500 steps) outgrows B = 400
        assert sum(1 for x in b[450:950] if x & 4) == 400


def test_pooled_loop_single_chain_is_the_reference_core():
    """The pooled loop at C = 1 is the single-chain warm-up: the metric at every window end is the reset core's."""
    rs = np.random.default_rng(7)
    T, d = 120, 5
    draws = rs.standard_normal((T, 1, d))
    grads = -draws + 0.05 * rs.standard_normal((T, 1, d))
    acc = rs.uniform(0.5, 1.0, (T, 1))
    sched = bj.build_schedule(T)
    run = o.run_pooled(draws, grads, acc, sched, max_rank=2)
    assert len(run.step_sizes) == T and len(run.metrics) == sum(1 for _, e in sched if e)
    core = o.ResetCore(d, 2, 1e-5, 2.0, o.buffer_size(T))
    for t, (st, e) in enumerate(sched):
        if st:
            core.update(draws[t], grads[t])
        if e:
            core.final()
            m = [m for m in run.metrics if m[0] == t][0]
            np.testing.assert_array_equal(m[1], core.sigma)


# ---- argument checks (no GPU needed) --------------------------------------------------------------------------------
def test_rejections_without_gpu():
    tgt = bj.targets.StdNormal(4)
    with pytest.raises(NotImplementedError):
        bj.window_adaptation_low_rank(bj.nuts, tgt, buffer_policy="accumulating")
    with pytest.raises(ValueError):
        bj.window_adaptation_low_rank(bj.nuts, tgt, buffer_policy="other")
    with pytest.raises(NotImplementedError):
        bj.window_adaptation_low_rank(bj.nuts, tgt, gradient_based_init=True)
    for r in (0, 17):
        with pytest.raises(ValueError):
            bj.window_adaptation_low_rank(bj.nuts, tgt, max_rank=r)
    with pytest.raises(ValueError):
        bj.window_adaptation_low_rank(bj.nuts, tgt, integrator=object())
    with pytest.raises(ValueError):
        bj.window_adaptation_low_rank(bj.mclmc, tgt)
    with pytest.raises(ValueError):
        bj.window_adaptation_low_rank(bj.hmc, tgt)   # no num_integration_steps
    with pytest.raises(ValueError):
        lra.schedule_bytes([(0, True)], 1)
