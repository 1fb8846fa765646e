"""MCLMC's tuner on the GPU (k_mclmc_tune, k_ess_chain and bjx_mclmc_find_l_and_step_size) against the float32 restatement
in oracle/mclmc_tuning.py.

* one tuning step, teacher-forced: state within close() of the oracle, success identical; the new step size, time,
  x_average, step_size_max and the streaming weight within 1e-5 relative, and the moment rows within close(), of the
  oracle's predictor and moment update fed with the device's own energy change; every warp size class, every built-in row target, a plug-in, all four
  tables, shared and per-chain metrics, mask 0 and 1, and the failure cases of the bounded target;
* the per-chain ESS against the float64 oracle/diagnostics on one-chain slices, and bit-identical to the pooled ESS kernel
  on one-chain handles;
* the native tuner: bit-identical for any stage-3 slice size, for two handles of C/2 chains with chain_offset, and for the
  plug-in diagonal Gaussian against the built-in target; it agrees with the oracle's tuner chain by chain;
* unsupported configurations and foreign kernels are rejected;
* the reference's statistical tests, every chain tuning on its own.
"""
import math

import numpy as np
import pytest
import torch

import blackjax_b200 as bj
from blackjax_b200 import _engine, _lib, plugin, targets as T
from blackjax_b200.adaptation import mclmc_adaptation as ma
from blackjax_b200.mcmc import integrators
from oracle import mclmc as om
from oracle import mclmc_tuning as ot
from oracle import prng as oprng
from oracle import targets as otargets
from oracle.diagnostics import effective_sample_size as oracle_ess
from test_gpu_parity import close, npy, tf, tk

pytestmark = pytest.mark.gpu
F = np.float32
TABLES = {"velocity_verlet": integrators.isokinetic_velocity_verlet, "mclachlan": integrators.isokinetic_mclachlan,
          "yoshida": integrators.isokinetic_yoshida, "omelyan": integrators.isokinetic_omelyan}


def _user_diag(s):
    inv_var = (1.0 / (np.asarray(s, np.float64) ** 2)).astype(F)
    return T.UserTarget(len(s), plugin.read_example("diag_gaussian"), inv_var, name="diag_gaussian")


def _bounded():
    return T.UserTarget(2, plugin.read_example("bounded_gaussian"), np.array([5.0], F), name="bounded_gaussian",
                        dense_metric=False, general_integrators=True)


def _targets(name, D, rs):
    if name == "diag":
        s = np.exp(rs.uniform(-0.5, 0.5, D))
        return T.DiagGaussian(s), otargets.DiagGaussian(s), 1.0
    if name == "funnel":
        return T.Funnel(D), otargets.Funnel(D), 0.3
    if name == "banana":
        return T.Banana(), otargets.Banana(), 0.5
    if name == "dense":
        A = rs.standard_normal((D, D)) / np.sqrt(D)
        P = (A @ A.T + np.eye(D)).astype(F)
        P = 0.5 * (P + P.T)
        return T.DenseGaussian(P), otargets.DenseGaussian(P), 1.0
    if name == "user_diag":
        s = np.exp(rs.uniform(-0.5, 0.5, D))
        return _user_diag(s), otargets.DiagGaussian(s), 1.0
    raise ValueError(name)


def _rel(a, b, rtol=1e-5):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    both_inf = np.isinf(a) & np.isinf(b) & (np.sign(a) == np.sign(b))
    ok = both_inf | (np.abs(a - b) <= rtol * np.maximum(np.abs(b), 1e-30))
    assert ok.all(), (a[~ok][:5], b[~ok][:5])


CASES = (  # (target, D, table, metric, mask)
    [("diag", D, "mclachlan", "shared", 1) for D in (2, 18, 70, 128, 256, 512, 1024)]
    + [("diag", 100, t, "per_chain", 1) for t in ("velocity_verlet", "yoshida", "omelyan")]
    + [("diag", 70, "mclachlan", "per_chain", 0), ("funnel", 256, "mclachlan", "shared", 1),
       ("banana", 2, "velocity_verlet", "shared", 1), ("dense", 70, "mclachlan", "per_chain", 1),
       ("user_diag", 128, "omelyan", "shared", 1), ("user_diag", 18, "mclachlan", "per_chain", 0)])


def _tune_both(tgt, otgt, state, imm, L, eps, adaptive, streaming, mask, table, step_key, C, D):
    """one teacher-forced tuning step on the device and in the oracle; returns (device outputs, oracle outputs)"""
    keys = oprng.split(step_key, C)
    k = ot.Constants(D)
    o = ot.tune_step(keys, state, otgt, imm, L, eps, adaptive, streaming, float(mask), TABLES[table], np.inf, k)
    eng = _engine.get_engine(tf(state[0]), tgt)
    eng.set_integrator(integrators.as_coefficients(TABLES[table]))
    eng.ensure_metric(tf(imm), diagonal_only=True)
    dst = [tf(x) for x in state]
    d_eps = tf(np.broadcast_to(eps, (C,)))
    d_ad = [tf(a) for a in adaptive]
    d_st = (tf(streaming[0]), tf(streaming[1]))
    ok = ma.tune_step_(eng, tk(step_key), dst, d_eps, float(L), np.inf, d_ad, d_st, mask)
    # the predictor and the moments in the oracle, fed with the device's own transition (the same rng keys through
    # k_mclmc_transition): the scalars are then held to 1e-5 without the rounding of the energy change's reductions
    st = bj.mcmc.hmc.IntegratorState(*(tf(x) for x in state))
    _, info = bj.mclmc.build_kernel(integrator=TABLES[table])(tk(oprng.split(keys, 2)[:, 0]), st, tgt, tf(imm), float(L),
                                                              tf(np.broadcast_to(eps, (C,))))
    torch.cuda.synchronize()
    success = npy(ok)
    eps_new, adaptive_new = ot.predictor(npy(info.energy_change), success, np.broadcast_to(eps, (C,)).astype(F), adaptive,
                                         k)
    weight = (F(mask) * success.astype(F) * eps_new).astype(F)
    streaming_new = ot.incremental_value_update(npy(dst[0]), streaming[0], streaming[1], weight)
    forced = (eps_new, adaptive_new, streaming_new)
    return (dst, d_eps, d_ad, d_st, ok), o, forced


@pytest.mark.parametrize("name, D, table, metric, mask", CASES)
def test_tune_step_matches_oracle(name, D, table, metric, mask):
    rs = np.random.default_rng(D * 11 + len(name) + len(table) + mask)
    C = 67
    tgt, otgt, scale = _targets(name, D, rs)
    q = (scale * rs.standard_normal((C, D))).astype(F)
    u = rs.standard_normal((C, D))
    u = (u / np.linalg.norm(u, axis=1, keepdims=True)).astype(F)
    logp, g = otgt(q)
    imm = np.exp(rs.uniform(-0.5, 0.5, (C, D) if metric == "per_chain" else D)).astype(F)
    eps = (rs.uniform(0.1, 0.4, C) * math.sqrt(D) * (0.2 if name == "funnel" else 1.0)).astype(F)
    L = F(math.sqrt(D))
    adaptive = (rs.uniform(0.5, 2.0, C).astype(F), rs.uniform(0.5, 2.0, C).astype(F),
                np.where(rs.uniform(size=C) < 0.5, np.inf, 2.0 * eps).astype(F))
    if mask:
        streaming = (rs.uniform(0.5, 3.0, C).astype(F), rs.standard_normal((C, 2, D)).astype(F))
    else:  # stage 1: no weight accumulated yet
        streaming = (np.zeros(C, F), np.zeros((C, 2, D), F))
    (dst, d_eps, d_ad, d_st, ok), (ost, oeps, oad, ost2, ook), (feps, fad, fst) = _tune_both(
        tgt, otgt, (q, u, logp, g), imm, L, eps, adaptive, streaming, mask, table, oprng.key(500 + D), C, D)
    assert np.array_equal(npy(ok), ook)
    close(npy(dst[0]), ost[0])
    close(npy(dst[1]), ost[1], scale=1.0 / math.sqrt(D))
    close(npy(dst[3]), ost[3])
    close(npy(dst[2]), ost[2], scale=max(float(np.max(np.abs(logp))), 1.0))
    _rel(npy(d_eps), feps)
    for a, b in zip(d_ad, fad):
        _rel(npy(a), b)
    _rel(npy(d_st[0]), fst[0])
    close(npy(d_st[1]), fst[1])  # total av + w x can cancel: held to 1e-5 of the row's scale


@pytest.mark.parametrize("table", ["mclachlan", "velocity_verlet"])
def test_tune_step_failures_on_the_bounded_target(table):
    """#969: step size 100 / 8 on the bounded target; failed chains keep their whole state, momentum included, and take
    step_size_max = 0.8 eps."""
    C = 64
    tgt, otgt = _bounded(), otargets.BoundedGaussian(2)
    init_keys = oprng.split(oprng.key(3), C)
    ostate = om.mclmc_init(np.zeros((C, 2), F), otgt, init_keys)
    eps = np.full(C, 100.0 if table == "mclachlan" else 8.0, F)
    adaptive = (np.zeros(C, F), np.zeros(C, F), np.full(C, np.inf, F))
    streaming = (np.ones(C, F), np.full((C, 2, 2), 0.25, F))
    (dst, d_eps, d_ad, d_st, ok), (ost, oeps, oad, ost2, ook), (feps, _, fst) = _tune_both(
        tgt, otgt, ostate, np.ones(2, F), F(1.0), eps, adaptive, streaming, 1, table, oprng.key(4), C, 2)
    ok = npy(ok)
    assert np.array_equal(ok, ook) and (~ok).any()
    for a, b in zip(dst, ostate):
        assert np.array_equal(npy(a)[~ok], np.asarray(b)[~ok])
    assert np.all(npy(d_ad[2])[~ok] == F(0.8) * eps[~ok])
    _rel(npy(d_eps), feps)
    close(npy(d_st[1]), fst[1])


@pytest.mark.parametrize("T_", [2, 3, 7, 100, 1000])
def test_ess_per_chain_matches_oracle(T_):
    rs = np.random.default_rng(T_)
    C, D = 6, 40
    x = np.empty((T_, C, D), np.float64)
    x[:, :, :15] = rs.standard_normal((T_, C, 15))
    z = np.zeros((C, 15))
    for t in range(T_):  # AR(1), phi = 0.99
        z = 0.99 * z + rs.standard_normal((C, 15))
        x[t, :, 15:30] = z
    x[:, :, 30:] = 1.5  # constant dimensions
    x = x.astype(F)
    eng = _engine.get_engine(tf(x[0]), T.StdNormal(D))
    ess = npy(bj.diagnostics.effective_sample_size(tf(x), T.StdNormal(D), per_chain=True))
    for c in range(C):
        want = np.atleast_1d(oracle_ess(x[:, c][None], chain_axis=0, sample_axis=1))
        assert np.all(ess[c, 30:] == 0) and np.all(want[30:] == 0)
        _rel(ess[c, :30], want[:30], rtol=1e-4)
    # the pooled kernel on a one-chain handle gives the same bits
    for c in range(C):
        ref = npy(bj.diagnostics.effective_sample_size(tf(x[:, c:c + 1]), T.StdNormal(D)))
        assert np.array_equal(ref, ess[c])
    del eng


def _tune_native(tgt, q0, key, num_steps=400, table="mclachlan", max_history_bytes=1 << 31, chain_offset=0, st=None,
                 **kw):
    st = bj.mclmc.init(q0, tgt, key) if st is None else st
    kernel = bj.mclmc.build_kernel(integrator=TABLES[table], chain_offset=chain_offset)
    return st, ma.mclmc_find_L_and_step_size(kernel, num_steps, st, key, tgt, max_history_bytes=max_history_bytes, **kw)


def test_native_tuner_bit_identity():
    D, C = 64, 96
    rs = np.random.default_rng(12)
    s = np.exp(rs.uniform(-1, 1, D))
    q0 = tf(rs.standard_normal((C, D)))
    key = tk(oprng.key(31))
    st, (fin, par, n) = _tune_native(T.DiagGaussian(s), q0, key)
    assert n == 400 // 10 * 3 + 40 // 3
    # stage 3 on slices of 5 chains
    _, (fin2, par2, _) = _tune_native(T.DiagGaussian(s), q0, key, max_history_bytes=40 * D * 4 * 5)
    # plug-in target
    _, (fin3, par3, _) = _tune_native(_user_diag(s), q0, key)
    torch.cuda.synchronize()
    for other_fin, other_par in ((fin2, par2), (fin3, par3)):
        for a, b in zip(list(fin) + list(par), list(other_fin) + list(other_par)):
            assert torch.equal(a, b)
    # two handles of C/2 chains with chain_offset
    halves = []
    for lo in (0, C // 2):
        sub = bj.mcmc.hmc.IntegratorState(*(t[lo:lo + C // 2].clone() for t in st))
        _, (f, p, _) = _tune_native(T.DiagGaussian(s), None, key, chain_offset=lo, st=sub)
        halves.append((f, p))
    torch.cuda.synchronize()
    for i in range(4):
        assert torch.equal(torch.cat([halves[0][0][i], halves[1][0][i]]), fin[i])
    for i in range(3):
        assert torch.equal(torch.cat([halves[0][1][i], halves[1][1][i]]), par[i])
    assert torch.isfinite(par.L).all() and (par.step_size > 0).all()


@pytest.mark.parametrize("diag", [True, False])
def test_native_tuner_matches_oracle(diag):
    """A short tune (num_steps = 20: two steps per stage, one readjustment) chain by chain against the oracle's tuner with
    per-chain keys.  The step count and the divergence flags agree exactly.  The tuned parameters are held to 10 %: each
    step size goes as xi^(-1/6) of an energy change that is a small difference of log-densities, so the last-bit
    differences of those reductions move it by a few percent within a step (up to 3 % seen); the teacher-forced tests
    above pin the arithmetic itself."""
    D, C = 8, 5
    rs = np.random.default_rng(3)
    s = np.exp(rs.uniform(-1, 1, D))
    q0 = rs.standard_normal((C, D)).astype(F)
    keys = oprng.split(oprng.key(77), C)
    st = bj.mclmc.init(tf(q0), T.DiagGaussian(s), tk(keys))
    n1, n2, r, _, _ = ma.stage_lengths(20, 0.1, 0.1, 0.1, diag)
    div = torch.empty(n1 + n2 + r, C, dtype=torch.uint8, device="cuda")
    fin, par, n = ma.mclmc_find_L_and_step_size(bj.mclmc.build_kernel(), 20, st, tk(keys), T.DiagGaussian(s),
                                                diagonal_preconditioning=diag, divergences=div)
    ostate = tuple(npy(t) for t in st)
    _, (oL, oeps, oimm), on, odiv = ot.find_L_and_step_size(keys, 20, ostate, otargets.DiagGaussian(s),
                                                            TABLES["mclachlan"], diagonal_preconditioning=diag)
    torch.cuda.synchronize()
    assert n == on and np.array_equal(npy(div).astype(bool), odiv)
    np.testing.assert_allclose(npy(par.step_size), oeps, rtol=0.1)
    np.testing.assert_allclose(npy(par.inverse_mass_matrix), oimm, rtol=0.1, atol=1e-4)
    np.testing.assert_allclose(npy(par.L), oL, rtol=0.1)


def test_unsupported_configurations_are_rejected():
    rs = np.random.default_rng(0)
    key = tk(oprng.key(0))
    kernel = bj.mclmc.build_kernel()
    for D in (1, 1028):
        q = tf(rs.standard_normal((8, D)))
        st = bj.mcmc.hmc.IntegratorState(q, q.clone(), tf(np.zeros(8)), q.clone())
        with pytest.raises(_lib.BjxError, match="error -2"):
            ma.mclmc_find_L_and_step_size(kernel, 100, st, key, T.StdNormal(D))
    # a dense Gaussian target beyond 128 dims
    tgt = T.DenseGaussian(np.eye(132, dtype=F))
    q = tf(rs.standard_normal((8, 132)))
    st = bj.mcmc.hmc.IntegratorState(q, q.clone(), tf(np.zeros(8)), q.clone())
    with pytest.raises(_lib.BjxError, match="error -2"):
        ma.mclmc_find_L_and_step_size(kernel, 100, st, key, tgt)
    # dense and low-rank metrics on the tuning step
    from blackjax_b200.mcmc.metrics import LowRankMetric
    D = 64
    q = tf(rs.standard_normal((8, D)))
    st = [q, q.clone(), tf(np.zeros(8)), q.clone()]
    for imm in (tf(np.broadcast_to(np.eye(D, dtype=F), (8, D, D))),
                LowRankMetric(torch.ones(D), torch.eye(D, 2), torch.full((2,), 2.0))):
        eng = _engine.get_engine(q, T.StdNormal(D))
        eng.ensure_metric(imm)
        z = torch.zeros(8, device="cuda")
        with pytest.raises(_lib.BjxError, match="error -2"):
            ma.tune_step_(eng, key, st, torch.ones(8, device="cuda"), 3.0, np.inf, (z, z.clone(), z.clone()), None, 0)
    with pytest.raises(TypeError):
        ma.mclmc_find_L_and_step_size(bj.hmc.build_kernel(), 100, st, key, T.StdNormal(D))


def _regression():
    rs = np.random.default_rng(42)
    x = rs.standard_normal((1000, 1)).astype(F)
    y = (3 * x[:, 0] + rs.standard_normal(1000)).astype(F)
    return T.LinearRegression(x, y)


def test_regression_posterior():
    """test_sampling.py:408-430 (run_mclmc :113-159): tune from (log_scale, coefs) = (1, 1), then 10000 steps; on every
    chain the mean scale is 1 +- 0.1 and the mean coefficient 3 +- 0.1."""
    tgt = _regression()
    C = 64
    key = tk(oprng.key(8))
    st, (fin, par, _) = _tune_native(tgt, tf(np.ones((C, 2))), key, num_steps=10000, diagonal_preconditioning=False)
    _, hist, _ = bj.sample_mclmc_native(tk(oprng.key(9)), fin, tgt, par.L, par.step_size, 10000,
                                        inverse_mass_matrix=par.inverse_mass_matrix, thin=10)
    h = npy(hist)
    assert np.all(np.abs(np.exp(h[..., 0]).mean(0) - 1.0) < 0.1)
    assert np.all(np.abs(h[..., 1].mean(0) - 3.0) < 0.1)


def test_preconditioning_direction_on_every_chain():
    """test_sampling.py:482-557 with 256 chains: D = 100, condition number 10, 20000 steps."""
    dim, kappa, C = 100, 10.0, 256
    eigs = np.logspace(-0.5 * np.log10(kappa), 0.5 * np.log10(kappa), dim)
    tgt = T.DiagGaussian(np.sqrt(eigs))
    rs = np.random.default_rng(2)
    q0 = tf(rs.standard_normal((C, dim)) * np.max(np.sqrt(eigs)))
    _, (_, par, _) = _tune_native(tgt, q0, tk(oprng.key(2)), num_steps=20000, diagonal_preconditioning=True)
    m2 = npy(par.inverse_mass_matrix).astype(np.float64) ** 2
    crit = np.abs((m2 / np.linalg.norm(m2, axis=1, keepdims=True)) @ (eigs / np.linalg.norm(eigs)) - 1)
    assert np.all(crit < 0.1), crit.max()


@pytest.mark.parametrize("table", ["mclachlan", "velocity_verlet"])
def test_convergence_from_large_step_size_on_the_bounded_target(table):
    """test_mclmc_nan_fix_969.py:168-176 with 256 chains: from step size 100, the final step sizes land in (0.1, 10).  The
    reference checks six keys; over 256 a few velocity Verlet chains shrink further, and they are the oracle's."""
    C = 256
    tgt = _bounded()
    key = tk(oprng.key(100))
    st = bj.mclmc.init(tf(np.zeros((C, 2))), tgt, key)
    kernel = bj.mclmc.build_kernel(integrator=TABLES[table])
    params = ma.MCLMCAdaptationState(math.sqrt(2.0), 100.0, 1.0)
    _, par, _ = ma.mclmc_find_L_and_step_size(kernel, 60, st, key, tgt, params=params, frac_tune1=1.0, frac_tune2=0.0,
                                              frac_tune3=0.0, diagonal_preconditioning=False)
    eps = npy(par.step_size)
    inside = (eps >= 0.1) & (eps <= 10.0)
    assert inside.mean() >= 0.98, eps[~inside]
    ck = oprng.fold_in(oprng.key(100), np.arange(C))
    ost = om.mclmc_init(np.zeros((C, 2), F), otargets.BoundedGaussian(2), ck)
    _, (_, oeps, _), _, _ = ot.find_L_and_step_size(ck, 60, ost, otargets.BoundedGaussian(2), TABLES[table],
                                                    frac_tune1=1.0, frac_tune2=0.0, frac_tune3=0.0,
                                                    diagonal_preconditioning=False,
                                                    params=(np.sqrt(F(2)), F(100), np.ones(2, F)))
    assert np.array_equal(inside, (oeps >= 0.1) & (oeps <= 10.0))
