"""CPU tests of the adjusted MCLMC / MAMS restatement (oracle/adjusted_mclmc.py): its trajectory and energy
difference against explicit compositions of the MCLMC oracle's integrator step, the key tree at n = 0, the step-count rules
(rescale, the Halton lengths), a long run on a small Gaussian (and the bias of unadjusted MCLMC at the same step size that
the adjustment removes), and the Python surface of blackjax_b200.adjusted_mclmc / adjusted_mclmc_dynamic without a
GPU."""
import math
import warnings

import numpy as np
import pytest
import torch

from oracle import adjusted_mclmc as oa
from oracle import mclmc as om
from oracle import prng as oprng
from oracle import targets as otargets

F = np.float32
MCLACHLAN = (0.1931833275037836, 0.5, 1.0 - 2 * 0.1931833275037836, 0.5, 0.1931833275037836)
VELOCITY_VERLET = (0.5, 1.0, 0.5)


def _state(C, D, target, seed):
    rs = np.random.default_rng(seed)
    q = rs.standard_normal((C, D)).astype(F)
    logp, g = target(q)
    return q, logp, g


@pytest.mark.parametrize("table", [VELOCITY_VERLET, MCLACHLAN])
def test_no_refresh_trajectory_is_n_integrator_steps(table):
    """With L_proposal_factor = inf the proposal is n compositions of the isokinetic step from the unit momentum of
    split(key)[0], and Delta = -logp_0 + logp_n - (sum of the steps' kinetic changes)."""
    C, D = 6, 5
    target = otargets.DiagGaussian(np.linspace(0.5, 2.0, D))
    q, logp, g = _state(C, D, target, 1)
    keys = oprng.split(oprng.key(7), C)
    n = np.array([0, 1, 2, 3, 5, 8], np.int32)
    eps = F(0.4)
    imm = np.linspace(0.8, 1.5, D).astype(F)
    new, info = oa.adjusted_mclmc_kernel(keys, (q, logp, g), target, imm, eps, n, table)
    u = om.unit_vector(oprng.split(keys, 2)[:, 0], D)
    np.testing.assert_array_equal(info.momentum, u)
    for c in range(C):
        qc, uc, lc, gc, kin = q[c:c + 1], u[c:c + 1], logp[c:c + 1], g[c:c + 1], F(0)
        for _ in range(n[c]):
            qc, uc, lc, gc, dk = om.isokinetic_step(qc, uc, lc, gc, target, np.sqrt(imm), eps, table)
            kin = F(kin + dk[0])
        np.testing.assert_array_equal(info.proposal[0][c], qc[0])
        np.testing.assert_array_equal(info.proposal[1][c], uc[0])
        assert info.delta[c] == F(F(-logp[c] + lc[0]) - kin)
        assert info.energy[c] == -lc[0]
    assert np.array_equal(info.num_integration_steps, n)


def test_zero_steps_accepts_with_the_integrator_key():
    """n = 0: the trajectory is the input state, Delta = 0, p_accept = 1, and the uniform is drawn from key_integrator."""
    C, D = 8, 3
    target = otargets.StdNormal(D)
    q, logp, g = _state(C, D, target, 2)
    keys = oprng.split(oprng.key(3), C)
    new, info = oa.adjusted_mclmc_kernel(keys, (q, logp, g), target, np.ones(D, F), F(0.5), 0, MCLACHLAN, F(1.0))
    assert np.all(info.acceptance_rate == 1) and info.is_accepted.all() and np.all(info.delta == 0)
    np.testing.assert_array_equal(info.uniform, oprng.uniform(oprng.split(keys, 2)[:, 1]))
    np.testing.assert_array_equal(new[0], q)
    # with n >= 1 the uniform comes from k_n instead
    _, info1 = oa.adjusted_mclmc_kernel(keys, (q, logp, g), target, np.ones(D, F), F(0.5), 2, MCLACHLAN)
    k = oprng.split(keys, 2)[:, 1]
    for _ in range(2):
        k = oprng.split(k, 2)[:, 1]
    np.testing.assert_array_equal(info1.uniform, oprng.uniform(k))


def test_partial_refresh_uses_the_step_keys():
    """A finite L_proposal_factor: step i refreshes with split(a_i)[0] and split(a_i)[1], L = factor * n * eps."""
    C, D, n = 4, 6, 2
    target = otargets.StdNormal(D)
    q, logp, g = _state(C, D, target, 4)
    keys = oprng.split(oprng.key(11), C)
    eps, fac = F(0.3), F(1.5)
    _, info = oa.adjusted_mclmc_kernel(keys, (q, logp, g), target, np.ones(D, F), eps, n, VELOCITY_VERLET, fac)
    L = F(fac * F(F(n) * eps))
    km = oprng.split(keys, 2)
    u, k = om.unit_vector(km[:, 0], D), km[:, 1]
    qq, ll, gg = q, logp, g
    for _ in range(n):
        ak = oprng.split(k, 2)
        a, k = ak[:, 0], ak[:, 1]
        r = oprng.split(a, 2)
        u = om.partial_refresh(u, r[:, 0], F(eps * F(0.5)), L)
        qq, u, ll, gg, _ = om.isokinetic_step(qq, u, ll, gg, target, np.ones(D, F), eps, VELOCITY_VERLET)
        u = om.partial_refresh(u, r[:, 1], F(eps * F(0.5)), L)
    np.testing.assert_array_equal(info.proposal[1], u)
    np.testing.assert_array_equal(info.proposal[0], qq)


def _floor_mean(s):
    """E[floor(U s)] for U ~ U(0, 1), exactly: (1/s) sum_{j=1}^{floor(s)} (s - j)."""
    m = int(math.floor(s))
    return sum(s - j for j in range(1, m + 1)) / s if s > 0 else 0.0


@pytest.mark.parametrize("mu", [1.0, 1.3, 2.0, 2.75, 3.5, 4.0, 6.2, 8.0, 10.5, 17.0, 31.3])
def test_rescale_gives_the_mean(mu):
    """round(U rescale(mu) + 0.5) and ceil(U rescale(mu)) both have mean mu (each is 1 + floor(U s) almost surely)."""
    s = float(oa.rescale(mu))
    np.testing.assert_allclose(1.0 + _floor_mean(s), mu, rtol=2e-6)
    # and a dense quadrature of the two rules themselves
    U = (np.arange(200000) + 0.5) / 200000
    np.testing.assert_allclose(np.mean(np.rint(U * s + 0.5)), mu, rtol=2e-4)
    np.testing.assert_allclose(np.mean(np.ceil(U * s)), mu, rtol=2e-4)


def test_halton_trajectory_lengths():
    """halton(t) = 0.5, 0.25, 0.75, 0.125, ...; with mu = 4, rescale = 7 and the lengths rint(0.5 + 7 h) are 4, 2, 6, 1."""
    np.testing.assert_array_equal(oa.halton_sequence(np.arange(6)), F([0.5, 0.25, 0.75, 0.125, 0.625, 0.375]))
    assert oa.rescale(4.0) == F(7.0)
    np.testing.assert_array_equal(oa.trajectory_length(np.arange(4), 4.0), [4, 2, 6, 1])
    from blackjax_b200.mcmc import adjusted_mclmc_dynamic as amd
    t = np.arange(64)
    np.testing.assert_array_equal(amd.halton_sequence(t), oa.halton_sequence(t))
    np.testing.assert_array_equal(amd.halton_sequence(torch.arange(64)).numpy(), oa.halton_sequence(t))
    for mu in (2.5, 4.0, 7.3):
        np.testing.assert_array_equal(amd.trajectory_length(t, mu), oa.trajectory_length(t, mu))
        np.testing.assert_array_equal(amd.trajectory_length(torch.arange(64), mu).numpy(), oa.trajectory_length(t, mu))


def test_step_rules():
    keys = oprng.split(oprng.key(5), 4000)
    n = oa.steps_randint(keys)
    assert n.min() == 1 and n.max() == 9
    u = oa.steps_uniform(keys, 8.0, min_steps=0)
    assert u.min() >= 0 and abs(u.mean() - 8.0) < 0.3
    assert oa.steps_uniform(keys, 0.7).min() == 1 and oa.steps_uniform(keys, 0.7, min_steps=0).max() == 0


SCALES = np.array([0.5, 1.0, 2.0, 4.0])


def _gaussian_run(kernel, T, seed=0):
    C, D = 512, len(SCALES)
    target = otargets.DiagGaussian(SCALES)
    rs = np.random.default_rng(seed)
    st = kernel.init((SCALES * rs.standard_normal((C, D))).astype(F), target)
    draws, accs = [], []
    step_keys = oprng.split(oprng.key(seed + 100), T)
    for t in range(T):
        st, acc = kernel.step(oprng.split(step_keys[t], C), st, target)
        draws.append(st[0] / SCALES)
        accs.append(acc)
    return np.stack(draws), np.mean(accs)


class _Adjusted:
    def __init__(self, eps, n):
        self.eps, self.n = F(eps), n

    def init(self, q, target):
        logp, g = target(q)
        return q, logp, g

    def step(self, keys, st, target):
        new, info = oa.adjusted_mclmc_kernel(keys, st, target, SCALES ** 2, self.eps, self.n, MCLACHLAN, F(1.0))
        return new, info.acceptance_rate.mean()


class _Unadjusted:
    def __init__(self, eps, L):
        self.eps, self.L = F(eps), F(L)

    def init(self, q, target):
        u = om.unit_vector(oprng.split(oprng.key(9), q.shape[0]), q.shape[1])
        logp, g = target(q)
        return q, u, logp, g

    def step(self, keys, st, target):
        new, _ = om.mclmc_kernel(keys, st, target, SCALES ** 2, self.L, self.eps, MCLACHLAN)
        return new, 1.0


# the step size of the GPU moment test (tests/test_gpu_adjusted_mclmc.py) on the same whitened problem: mean acceptance
# 0.6 - 0.8, and unadjusted MCLMC at the same step size (L = 4 eps) underestimates the variance by about 12 %
EPS = 4.0


def test_long_run_recovers_gaussian_moments_and_removes_mclmc_bias():
    x, acc = _gaussian_run(_Adjusted(EPS, 4), 240)
    x = x[40:].reshape(-1, len(SCALES))
    assert 0.6 < acc < 0.85, acc
    assert np.all(np.abs(x.mean(0)) < 0.06), x.mean(0)
    assert np.all(np.abs(x.var(0) - 1.0) < 0.08), x.var(0)
    y, _ = _gaussian_run(_Unadjusted(EPS, EPS * 4), 240)
    y = y[40:].reshape(-1, len(SCALES))
    assert np.mean(y.var(0)) < 0.92, y.var(0)  # the integrator's bias, which the Metropolis correction removes


def test_python_surface_without_gpu():
    import inspect

    import blackjax_b200 as bj
    from blackjax_b200.mcmc import adjusted_mclmc as am
    from blackjax_b200.mcmc import adjusted_mclmc_dynamic as amd
    for mu in (1.0, 2.5, 8.0, 13.7):
        assert am.rescale(mu) == oa.rescale(mu)
    with pytest.raises(ValueError, match="Either `num_integration_steps` or `integration_steps_params`"):
        bj.adjusted_mclmc(bj.targets.StdNormal(4), 0.5)
    with pytest.warns(DeprecationWarning, match="`num_integration_steps` is deprecated"):
        bj.adjusted_mclmc(bj.targets.StdNormal(4), 0.5, num_integration_steps=3, integration_steps_params=(4,))
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        alg = bj.adjusted_mclmc(bj.targets.StdNormal(4), 0.5, num_integration_steps=3)
    assert list(inspect.signature(alg.step).parameters) == ["rng_key", "state"]
    assert list(inspect.signature(bj.adjusted_mclmc.build_kernel()).parameters) == [
        "rng_key", "state", "logdensity_fn", "step_size", "integration_steps_params", "inverse_mass_matrix",
        "L_proposal_factor"]
    assert list(inspect.signature(bj.adjusted_mclmc_dynamic.build_kernel()).parameters) == [
        "rng_key", "state", "logdensity_fn", "step_size", "L_proposal_factor", "inverse_mass_matrix",
        "integration_steps_params"]
    assert list(inspect.signature(bj.adjusted_mclmc_dynamic.init).parameters) == [
        "position", "logdensity_fn", "random_generator_arg"]
    assert am.steps_argument(3) == 3 and am.steps_argument(7.2) == 8 and am.steps_argument(0) == 0
    with pytest.raises(ValueError):
        am.steps_argument(-1)
    fixed = amd.make_random_trajectory_length_fn(False)
    assert fixed(None, 3.2) == 4 and fixed(None, 0.3) == 1
    assert amd.make_random_trajectory_length_fn(True).device_rule == (2, 1)
    assert amd.make_random_trajectory_length_fn(True, min_steps=0).device_rule == (2, 0)
