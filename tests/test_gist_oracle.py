"""GIST on the CPU: the oracle (oracle/gist.py) against the reference's known answers, the Python surface, and the sm_90a
compile of the GIST kernels (no stack frame, no spills).  No GPU is needed."""
import inspect
import os

import numpy as np
import pytest

import blackjax_b200 as bj
from oracle import gist as og
from oracle import hmc as ohmc
from oracle import prng
from oracle import targets as otargets
from test_kernel_spills import INSTANCES, NVCC, WITH_CSRC, assert_entries_clean, ptxas_log

F = np.float32


def rollout_states(target, metric, q, p, g, eps, n):
    """The states after 1..n integrator steps (the reference's rollout buffer)."""
    out = []
    for _ in range(n):
        q, p, _, g = ohmc.integrator_step(target, metric, q, p, g, eps)
        out.append((q, p, g))
    return out


# ---- trajectory length --------------------------------------------------------------------------------------------------
def test_quarter_period_uturn_anchor_1d():
    """1-D standard normal from (theta, rho) = (0, 1): theta_t = sin t, rho_t = cos t, and the no-return dot sin t cos t first
    turns negative just after a quarter period, t = pi / 2 (test_gist_trajectory_length.py's anchor)."""
    tgt, metric = otargets.StdNormal(1), ohmc.Metric(np.ones(1, F))
    for h in (0.1, 0.05, 0.2):
        q, p = np.zeros((1, 1), F), np.ones((1, 1), F)
        _, g = tgt(q)
        u = og.num_steps_to_uturn(tgt, metric, q, p, g, F(h), 1024)
        assert int(u[0]) == int(np.floor(np.pi / 2 / h)) + 1


def test_psi_zero_closed_form():
    """psi = 0: lo = 1 and width = U (eq. 34)."""
    u = np.arange(1, 50)
    lo, w = og.step_distribution(u, 0.0)
    assert (lo == 1).all() and (w == u).all()
    lo, w = og.step_distribution(u, 0.5)
    assert (lo == np.maximum(1, u // 2)).all() and (w == u - lo + 1).all()


def test_raw_momentum_pairing_not_velocity():
    """The no-return dot pairs the displacement with the raw momentum rho, not M^-1 rho: under a metric that rotates the
    velocity away from rho the two criteria stop at different steps, and the oracle follows the raw one."""
    D = 2
    tgt = otargets.StdNormal(D)
    imm = np.array([[1.0, 0.9], [0.9, 1.0]], F)
    metric = ohmc.Metric(imm)
    q = np.zeros((1, D), F)
    p = np.array([[1.0, -0.8]], F)
    _, g = tgt(q)
    u = int(og.num_steps_to_uturn(tgt, metric, q, p, g, F(0.05), 4096)[0])
    states = rollout_states(tgt, metric, q, p, g, F(0.05), u)
    raw = [float(np.sum((s[0] - q) * s[1])) for s in states]
    assert all(d >= 0 for d in raw[:-1]) and raw[-1] < 0
    vel = [float(np.sum((s[0] - q) * metric.velocity(s[1]))) for s in states]
    assert any(v < 0 for v in vel[:-1]) or vel[-1] >= 0  # the velocity pairing would decide elsewhere


def test_dense_metric_uturn_counts_match_whitened_ground_truth():
    """Affine equivariance: U under (target, dense metric) equals U of the whitened problem under the identity metric."""
    rs = np.random.default_rng(0)
    D, C = 4, 32
    A = rs.standard_normal((D, D))
    cov = (A @ A.T / D + np.eye(D)).astype(np.float64)
    L = np.linalg.cholesky(cov)
    tgt = otargets.DenseGaussian(np.linalg.inv(cov))
    metric = ohmc.Metric(cov.astype(F))
    z = rs.standard_normal((C, D))
    q = (z @ L.T).astype(F)
    keys = prng.split(prng.key(3), C)
    p = metric.sample_momentum(keys, D)
    _, g = tgt(q)
    u = og.num_steps_to_uturn(tgt, metric, q, p, g, F(0.1), 1024)
    wt, wm = otargets.StdNormal(D), ohmc.Metric(np.ones(D, F))
    qw = np.linalg.solve(L, q.T.astype(np.float64)).T.astype(F)
    pw = (p.astype(np.float64) @ L).astype(F)
    _, gw = wt(qw)
    uw = og.num_steps_to_uturn(wt, wm, qw, pw, gw, F(0.1), 1024)
    assert (np.abs(u - uw) <= 1).all() and (u == uw).mean() > 0.9


def test_max_num_steps_used_as_is():
    tgt, metric = otargets.StdNormal(1), ohmc.Metric(np.ones(1, F))
    q, p = np.zeros((1, 1), F), np.ones((1, 1), F)
    _, g = tgt(q)
    for cap in (1, 3, 15):
        assert int(og.num_steps_to_uturn(tgt, metric, q, p, g, F(0.1), cap)[0]) == cap


def test_reintegration_bit_identical_to_rollout_state():
    rs = np.random.default_rng(1)
    D, C = 5, 8
    tgt, metric = otargets.Funnel(D), ohmc.Metric(np.exp(rs.uniform(-0.5, 0.5, D)).astype(F))
    q = (0.5 * rs.standard_normal((C, D))).astype(F)
    p = rs.standard_normal((C, D)).astype(F)
    logp, g = tgt(q)
    states = rollout_states(tgt, metric, q, p, g, F(0.1), 12)
    steps = np.arange(C) % 12 + 1
    q1, p1, _, g1 = og.integrate_per_chain(tgt, metric, q, p, logp, g, F(0.1), steps)
    for c in range(C):
        k = steps[c] - 1
        assert np.array_equal(q1[c], states[k][0][c]) and np.array_equal(p1[c], states[k][1][c])
        assert np.array_equal(g1[c], states[k][2][c])


def test_no_return_rejection_and_absurd_step_size():
    rs = np.random.default_rng(2)
    D, C = 3, 200
    tgt = otargets.StdNormal(D)
    q = rs.standard_normal((C, D)).astype(F)
    st = ohmc.init(q, tgt)
    keys = prng.split(prng.key(5), C)
    _, info = og.gist_kernel(keys, st, tgt, F(0.3), np.ones(D, F), path_fraction=0.9)
    rej = info["rejected"]
    L, N = info["num_integration_steps"], info["reverse"]
    lo_r, _ = og.step_distribution(N, 0.9)
    assert (rej == ~((L >= lo_r) & (L <= N))).all()
    assert rej.any() and not info["is_accepted"][rej].any() and (info["acceptance_rate"][rej] == 0).all()
    new, info = og.gist_kernel(keys, st, tgt, F(1e4), np.ones(D, F))
    assert not info["is_accepted"].any() and np.array_equal(new[0], q)


# ---- step size ----------------------------------------------------------------------------------------------------------
def test_step_size_final_halving_and_criteria():
    """On a Gaussian the energy error grows with the step size: a tiny initial step expands (v = 1) and reports one step
    back from the first trial that stops expanding; a huge one halves (v = -1)."""
    rs = np.random.default_rng(4)
    D, C = 2, 64
    tgt, metric = otargets.StdNormal(D), ohmc.Metric(np.ones(D, F))
    q = rs.standard_normal((C, D)).astype(F)
    logp, g = tgt(q)
    p = rs.standard_normal((C, D)).astype(F)
    log_a, log_b = np.full(C, np.log(F(0.2)), F), np.full(C, np.log(F(0.8)), F)
    for crit in (False, True):
        j, ex = og.select_step_index(tgt, metric, q, p, logp, g, F(1e-3), log_a, log_b, 1, 30, crit)
        assert not ex.any() and (j > 0).all()
        # the trial at j + 1 is the first that did not expand: restated directly
        for c in range(4):
            def ell(jj):
                eps = F(1e-3) * F(2.0 ** jj)
                q1, p1, lp1, _ = ohmc.static_integration(tgt, metric, q[c:c + 1], p[c:c + 1], logp[c:c + 1], g[c:c + 1],
                                                         eps, 1)
                return float(og.safe_energy_diff(-logp[c] + metric.kinetic_energy(p[c:c + 1]),
                                                 -lp1 + metric.kinetic_energy(-p1))[0])
            small = (lambda x: abs(x) < abs(log_b[c])) if not crit else (lambda x: x >= log_b[c])
            assert small(ell(int(j[c]))) and not small(ell(int(j[c]) + 1))
        j, ex = og.select_step_index(tgt, metric, q, p, logp, g, F(50.0), log_a, log_b, 1, 30, crit)
        assert not ex.any() and (j < 0).all()


def test_search_exhausted_and_reversibility_force_rejection():
    rs = np.random.default_rng(5)
    D, C = 3, 256
    tgt = otargets.StdNormal(D)
    st = ohmc.init(rs.standard_normal((C, D)).astype(F), tgt)
    keys = prng.split(prng.key(6), C)
    _, info = og.gist_kernel(keys, st, tgt, F(1e-4), np.ones(D, F), instance="step_size", max_search_steps=0)
    assert info["rejected"].all() and not info["is_accepted"].any() and (info["forward"] == 0).all()
    _, info = og.gist_kernel(keys, st, tgt, F(0.5), np.ones(D, F), instance="step_size")
    irrev = (info["forward"] != info["reverse"]) & ~info["rejected"]
    assert irrev.any() and not info["is_accepted"][irrev].any()
    ok = info["is_accepted"]
    assert ok.any() and (info["forward"][ok] == info["reverse"][ok]).all()
    np.testing.assert_array_equal(info["step_size"], (F(0.5) * np.ldexp(F(1.0), info["forward"])).astype(F))


@pytest.mark.parametrize("instance", ["trajectory_length", "step_size"])
def test_stationarity_from_exact_draws(instance):
    """Exact draws of a small Gaussian stay distributed as the target after a few transitions (many oracle chains)."""
    rs = np.random.default_rng(7)
    D, C, T_ = 2, 4000, 3
    s = np.array([1.0, 2.0])
    tgt = otargets.DiagGaussian(s)
    q = (rs.standard_normal((C, D)) * s).astype(F)
    st = ohmc.init(q, tgt)
    for t in range(T_):
        keys = prng.split(prng.fold_in(prng.key(8), t), C)
        st, info = og.gist_kernel(keys, st, tgt, F(0.4), np.ones(D, F), instance=instance)
        assert info["is_accepted"].mean() > 0.3
    x = st[0].astype(np.float64)
    se = s / np.sqrt(C)
    assert (np.abs(x.mean(0)) < 5 * se).all()
    assert (np.abs(x.var(0) / s ** 2 - 1) < 5 * np.sqrt(2.0 / C)).all()


# ---- the Python surface -------------------------------------------------------------------------------------------------
def test_api_surface():
    sig = inspect.signature(bj.gist_trajectory_length.differentiable)
    assert list(sig.parameters)[:3] == ["logdensity_fn", "inverse_mass_matrix", "step_size"]
    assert sig.parameters["path_fraction"].default == 0.5 and sig.parameters["max_num_steps"].default == 1024
    assert sig.parameters["divergence_threshold"].default == 1000
    sig = inspect.signature(bj.gist_step_size.differentiable)
    assert list(sig.parameters)[:4] == ["logdensity_fn", "inverse_mass_matrix", "initial_step_size",
                                        "num_integration_steps"]
    assert sig.parameters["criterion"].default == "symmetric" and sig.parameters["max_search_steps"].default == 10
    kern = inspect.signature(bj.gist_step_size.build_kernel())
    assert list(kern.parameters) == ["rng_key", "state", "logdensity_fn", "initial_step_size", "inverse_mass_matrix",
                                     "num_integration_steps"]
    kern = inspect.signature(bj.gist_trajectory_length.build_kernel())
    assert list(kern.parameters) == ["rng_key", "state", "logdensity_fn", "step_size", "inverse_mass_matrix"]
    with pytest.raises(ValueError):
        bj.gist_step_size.build_kernel(criterion="neither")
    with pytest.raises(ValueError):
        bj.gist_step_size(None, None, 0.1, criterion="neither")
    from blackjax_b200.mcmc import composed
    assert {"GISTState", "GISTInfo", "init", "build_kernel"} <= set(composed.__all__)
    assert composed.trajectory_length.GISTTrajectoryLengthInfo._fields[-3:] == (
        "num_steps_to_uturn_forward", "num_steps_to_uturn_reverse", "is_no_return_rejected")
    assert composed.step_size.GISTStepSizeInfo._fields[-4:] == ("step_index", "reverse_step_index", "search_exhausted",
                                                                "step_size")


# ---- sm_90a compile -----------------------------------------------------------------------------------------------------
GIST_KERNELS = (("k_gist_transition", "Params, const uint32_t*, const float*, const float*, const float*, float*, float*, "
                                      "float*, GistArgs"),
                ("k_gist_chains", "Params, float*, float*, float*, GistArgs"))
@pytest.mark.skipif(not os.path.exists(NVCC), reason="needs nvcc")
def test_gist_kernels_compile_without_spills(tmp_path):
    lines = ['#include "bjx_kernels.cuh"', "namespace bjx {"]
    for row, tk in INSTANCES:
        for gen in ("false", "true"):
            for name, params in GIST_KERNELS:
                lines.append(f"template __global__ void {name}<{row}, {tk}, false, {gen}>({params});")
    log = ptxas_log(tmp_path, "\n".join(lines + ["}"]) + "\n", WITH_CSRC)
    assert_entries_clean(log, ("k_gist_",), 4 * len(INSTANCES))
