"""CPU tests of the MCLMC restatement (oracle/mclmc.py) against the reference's own known-answer tests
(tests/mcmc/test_integrators.py:225-349, tests/mcmc/test_mclmc_nan_fix_969.py:82-119), and the Python-side argument
handling of blackjax_b200.mclmc."""
import math

import numpy as np
import pytest
import torch

from oracle import mclmc as om
from oracle import prng as oprng
from oracle import targets as otargets

F = np.float32
TABLES = {"velocity_verlet": (0.5, 1.0, 0.5),
          "mclachlan": (0.1931833275037836, 0.5, 1.0 - 2 * 0.1931833275037836, 0.5, 0.1931833275037836)}
_b1y, _a1y = 0.11888010966548, 0.29619504261126
TABLES["yoshida"] = (_b1y, _a1y, 0.5 - _b1y, 1.0 - 2.0 * _a1y, 0.5 - _b1y, _a1y, _b1y)
_b1o, _a1o, _b2o, _a2o = 0.08398315262876693, 0.2539785108410595, 0.6822365335719091, -0.03230286765269967
_b3o, _a3o = 0.5 - _b1o - _b2o, 1.0 - 2.0 * (_a1o + _a2o)
TABLES["omelyan"] = (_b1o, _a1o, _b2o, _a2o, _b3o, _a3o, _b3o, _a2o, _b2o, _a1o, _b1o)


@pytest.mark.parametrize("dims", [3, 5])
def test_esh_momentum_update(dims):
    """The stable update equals the naive equation 16 of Robnik et al. (2023) (test_integrators.py:225-257)."""
    step_size = 1e-3
    k0, k1 = oprng.split(oprng.key(62), 2)
    gradient = oprng.uniform(k0, (dims,)).astype(np.float64)
    momentum = oprng.uniform(k1, (dims,)).astype(np.float64)
    momentum /= np.linalg.norm(momentum)
    gn = np.linalg.norm(gradient)
    gh = gradient / gn
    delta = step_size * gn / (dims - 1)
    naive = (momentum + gh * (np.sinh(delta) + np.dot(gh, momentum * (np.cosh(delta) - 1)))) / (
        np.cosh(delta) + np.dot(gh, momentum * np.sinh(delta)))
    new, _ = om.esh_update(momentum[None].astype(F), gradient[None].astype(F), np.ones(dims, F), F(step_size))
    np.testing.assert_array_almost_equal(new[0], naive)


def _cov_target(cov):
    return otargets.DenseGaussian(np.linalg.inv(np.asarray(cov, np.float64)).astype(F))


def _initial(dim, target):
    k0, k1 = oprng.split(oprng.key(4263456), 2)
    q = oprng.normal(k0, (dim,))[None]
    u = om.unit_vector(k1[None], dim)
    logp, g = target(q)
    return q, u, logp, g


def test_isokinetic_velocity_verlet_is_the_explicit_composition():
    """test_integrators.py:259-310: one isokinetic velocity Verlet step = op1(1/2) -> op2(1) -> op1(1/2)."""
    target = _cov_target([[1.0, 0.5, 0.1], [0.5, 2.0, -0.1], [0.1, -0.1, 3.0]])
    q, u, logp, g = _initial(3, target)
    eps, one = F(1e-4), np.ones(3, F)
    q1, u1, logp1, g1, kc = om.isokinetic_step(q, u, logp, g, target, one, eps, TABLES["velocity_verlet"])
    u_, k0 = om.esh_update(u, g, one, eps * F(0.5))
    q_ = om.position_update(q, u_, one, eps)
    logp_, g_ = target(q_)
    u_, k1 = om.esh_update(u_, g_, one, eps * F(0.5))
    for a, b in ((q1, q_), (u1, u_), (logp1, logp_), (g1, g_)):
        np.testing.assert_allclose(a, b, rtol=1e-6)
    np.testing.assert_almost_equal(kc, k0 + k1)


@pytest.mark.parametrize("table", list(TABLES))
def test_isokinetic_integrator_conserves_energy(table):
    """test_integrators.py:312-349: 15 steps of 1e-4 on a correlated 2-D Gaussian, energy change within 1e-3."""
    target = _cov_target([[1.0, 0.5], [0.5, 2.0]])
    q, u, logp, g = _initial(2, target)
    logp_init, kc = logp, None
    for _ in range(15):
        q, u, logp, g, kc = om.isokinetic_step(q, u, logp, g, target, np.ones(2, F), F(1e-4), TABLES[table])
    energy_change = kc[0] + (logp[0] - logp_init[0])
    assert abs(energy_change) < 1e-3


def _bounded_kernel(seed, table, step_size):
    target = otargets.BoundedGaussian(2)
    init_key, step_key = oprng.split(oprng.key(seed), 2)
    state = om.mclmc_init(np.zeros((1, 2), F), target, init_key[None])
    return om.mclmc_kernel(step_key[None], state, target, np.ones(2, F), F(1.0), F(step_size), TABLES[table])


def test_nan_fix_case1_mclachlan_reverts_and_flags():
    """test_mclmc_nan_fix_969.py:82-96: mclachlan, step size 100, key(0) overshoots the box."""
    (q, u, logp, g), info = _bounded_kernel(0, "mclachlan", 100.0)
    assert not info.nonans[0]
    assert np.isfinite(logp[0]) and np.all(np.isfinite(q)) and np.all(q == 0)
    assert info.energy_change[0] == 0 and info.kinetic_change[0] == 0
    np.testing.assert_allclose(np.linalg.norm(u[0]), 1.0, rtol=1e-6)


def test_nan_fix_case2_eight_seeds_all_flagged():
    """test_mclmc_nan_fix_969.py:99-119: velocity Verlet, step size 8, seeds 0..7 -- NaN log-density, all reverted."""
    for seed in range(8):
        (q, u, logp, g), info = _bounded_kernel(seed, "velocity_verlet", 8.0)
        assert not info.nonans[0], seed
        assert np.isfinite(logp[0]), seed


def test_high_energy_cutoff_reverts():
    """handle_high_energy (mclmc.py:257-281): |energy_change| above the cutoff keeps the state, momentum from the cutoff key."""
    target = otargets.StdNormal(8)
    rs = np.random.default_rng(0)
    q = rs.standard_normal((16, 8)).astype(F)
    keys = oprng.split(oprng.key(3), 16)
    state = om.mclmc_init(q, target, keys)
    _, free = om.mclmc_kernel(keys, state, target, np.ones(8, F), F(3.0), F(2.0), TABLES["mclachlan"])
    cutoff = float(np.median(np.abs(free.energy_change)))
    (q1, u1, logp1, _), info = om.mclmc_kernel(keys, state, target, np.ones(8, F), F(3.0), F(2.0), TABLES["mclachlan"],
                                               cutoff=cutoff)
    high = np.abs(free.energy_change) > F(cutoff)
    assert high.any() and (~high).any()
    assert np.array_equal(q1[high], q[high]) and np.all(info.energy_change[high] == 0) and np.all(info.nonans)
    np.testing.assert_array_equal(u1[high], om.unit_vector(oprng.split(keys, 3)[:, 1], 8)[high])


def test_python_surface_without_gpu():
    import blackjax_b200 as bj
    from blackjax_b200.mcmc import integrators, mclmc
    assert integrators.as_coefficients(integrators.isokinetic_mclachlan) == integrators.mclachlan
    assert integrators.as_coefficients("isokinetic_omelyan") == integrators.omelyan
    assert mclmc.energy_cutoff(100, math.inf, 5e-4) == math.inf
    assert mclmc.energy_cutoff(100, 2.0, 5e-4) == float(np.sqrt(F(100 * (2.0 * 5e-4))))
    with pytest.raises(ValueError, match="more than 1 dimension"):
        bj.mclmc.init(torch.zeros(4, 1), bj.targets.StdNormal(1), torch.zeros(2, dtype=torch.uint32))
    assert set(bj.mcmc.mclmc.MCLMCInfo._fields) == {"logdensity", "kinetic_change", "energy_change", "nonans"}
