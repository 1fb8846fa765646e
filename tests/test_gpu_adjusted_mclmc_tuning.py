"""Adjusted MCLMC's tuner on the GPU (k_amclmc_tune and bjx_adjusted_mclmc_find_l_and_step_size) against the float32
restatement in oracle/adjusted_mclmc_tuning.py.

* one tuning step, teacher-forced: step counts and success flags exact; the state within close() of the oracle; the DA
  fields, eps, L, the streaming total and moments within 1e-5 of the oracle's update fed with the device's own transition
  (the same keys through k_amclmc_transition), where reductions round differently;
* the revert path on the bounded target;
* the native tuner: bit-identical across stage-3 slice sizes and for two handles of C/2 chains with chain_offset, and
  against the oracle's tuner chain by chain;
* the reference's own tests on every chain of a batch, and the tuned parameters feeding the samplers;
* rejections.
"""
import math

import numpy as np
import pytest
import torch

import blackjax_b200 as bj
from blackjax_b200 import _engine, _lib, plugin, targets as T
from blackjax_b200.adaptation import adjusted_mclmc_adaptation as ama
from blackjax_b200.mcmc import adjusted_mclmc_dynamic as amd
from blackjax_b200.mcmc import integrators
from oracle import adjusted_mclmc as ao
from oracle import adjusted_mclmc_tuning as at
from oracle import prng as oprng
from oracle import targets as otargets
from oracle.adaptation import da_init
from test_gpu_parity import close, npy, tf, tk

pytestmark = pytest.mark.gpu
F = np.float32
TABLES = {"velocity_verlet": integrators.isokinetic_velocity_verlet, "mclachlan": integrators.isokinetic_mclachlan,
          "yoshida": integrators.isokinetic_yoshida, "omelyan": integrators.isokinetic_omelyan}
RULES = {"static": (None, ("static", None)), "randint": ((_lib.AMCLMC_STEPS_RANDINT, 0), ("randint", 0)),
         "uniform": ((_lib.AMCLMC_STEPS_UNIFORM, 1), ("uniform", 1))}


def _user_diag(s):
    inv_var = (1.0 / (np.asarray(s, np.float64) ** 2)).astype(F)
    return T.UserTarget(len(s), plugin.read_example("diag_gaussian"), inv_var, name="diag_gaussian")


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
    ok = (a == b) | (np.abs(a - b) <= rtol * np.maximum(np.abs(b), 1e-30))
    assert ok.all(), (a[~ok][:5], b[~ok][:5])


CASES = (  # (target, D, table, metric, mask, fix_L, rule)
    [("diag", D, "mclachlan", "shared", 1, True, "uniform") for D in (2, 18, 128, 512, 1024)]
    + [("diag", 100, t, "per_chain", 1, False, "randint") for t in ("velocity_verlet", "yoshida", "omelyan")]
    + [("diag", 70, "mclachlan", "per_chain", 0, True, "static"), ("funnel", 256, "mclachlan", "shared", 0, True, "uniform"),
       ("banana", 2, "velocity_verlet", "shared", 1, False, "static"), ("dense", 70, "mclachlan", "per_chain", 1, True,
                                                                         "randint"),
       ("user_diag", 128, "omelyan", "shared", 0, True, "uniform"), ("user_diag", 18, "mclachlan", "per_chain", 1, False,
                                                                       "static"),
       ("diag", 1024, "mclachlan", "per_chain", 0, True, "static"), ("diag", 600, "yoshida", "shared", 0, False,
                                                                       "uniform")])


@pytest.mark.parametrize("name, D, table, metric, mask, fix_L, rule", CASES)
def test_tune_step_matches_oracle(name, D, table, metric, mask, fix_L, rule):
    rs = np.random.default_rng(D * 13 + len(name) + len(table) + mask)
    C = 67
    tgt, otgt, scale = _targets(name, D, rs)
    q = (scale * rs.standard_normal((C, D))).astype(F)
    logp, g = otgt(q)
    rga = oprng.split(oprng.key(D), C)
    imm = np.exp(rs.uniform(-0.5, 0.5, (C, D) if metric == "per_chain" else D)).astype(F)
    eps = (rs.uniform(0.05, 0.3, C) * math.sqrt(D) * (0.2 if name == "funnel" else 1.0)).astype(F)
    L = (eps * rs.uniform(1.2, 4.0, C)).astype(F)
    da = tuple(np.broadcast_to(np.asarray(x, F), (C,)).copy() for x in da_init(eps))
    da = (da[0], rs.uniform(-1, 0, C).astype(F), np.full(C, 3.0, F), rs.uniform(-0.1, 0.1, C).astype(F), da[4])
    streaming = ((rs.uniform(0.5, 3.0, C).astype(F), rs.standard_normal((C, 2, D)).astype(F)) if not mask else
                 (np.zeros(C, F), np.zeros((C, 2, D), F)))
    device_rule, kind = RULES[rule]
    step_key = oprng.key(700 + D)
    keys = oprng.split(step_key, C)
    state = (q, logp, g) + ((rga,) if device_rule else ())
    # the device
    eng = _engine.get_engine(tf(q), tgt)
    eng.set_integrator(integrators.as_coefficients(TABLES[table]))
    eng.ensure_metric(tf(imm), diagonal_only=True)
    dst = [tf(x) for x in (q, logp, g)] + ([tk(rga)] if device_rule else [])
    d_eps, d_L, d_da = tf(eps), tf(L), tf(np.stack(da, 1))
    d_st = (tf(streaming[0]), tf(streaming[1]))
    d_count = tf(np.zeros(C, F))
    ok, steps = ama.tune_step_(eng, tk(step_key), dst, d_eps, d_L, d_da, d_st, d_count, mask, fix_L, 0.65,
                               device_rule=device_rule)
    # the device's own transition with the same keys and step counts, fed to the oracle's update
    n_dev = npy(steps)
    avg = (L / eps).astype(F)
    n_o, rep = at.num_steps_of(kind, avg, rga)
    st = bj.mcmc.hmc.HMCState(*(tf(x) for x in (q, logp, g)))
    new, info = bj.adjusted_mclmc.build_kernel(integrator=TABLES[table])(tk(keys), st, tgt, tf(eps), (tf(n_o),),
                                                                         tf(imm))
    torch.cuda.synchronize()
    assert np.array_equal(n_dev, n_o)
    new_np = tuple(npy(x) for x in new) + ((oprng.split(rga, 2)[:, 1],) if device_rule else ())
    dev_info = ao.Info(acceptance_rate=npy(info.acceptance_rate))
    o = at.tune_step(kind, keys, state, otgt, imm, eps, L, da, streaming, float(mask), fix_L, 0.65, TABLES[table],
                     info=(new_np, dev_info, n_o, rep))
    # and the oracle's own transition
    o_full = at.tune_step(kind, keys, state, otgt, imm, eps, L, da, streaming, float(mask), fix_L, 0.65, TABLES[table])
    assert np.array_equal(npy(ok), o_full[5])
    # the state against the oracle's handle_nans of the device's own transition; against the oracle's transition where
    # the Metropolis decision agrees (a uniform within the last bits of exp(Delta) can flip it at large D)
    close(npy(dst[0]), o[0][0])
    close(npy(dst[2]), o[0][2])
    close(npy(dst[1]), o[0][1], scale=max(float(np.max(np.abs(logp))), 1.0))
    o_acc = at.transition(kind, keys, state, otgt, imm, eps, L, TABLES[table])[1].is_accepted
    same = npy(info.is_accepted).astype(bool) == o_acc
    assert (~same).sum() <= 1
    close(npy(dst[0])[same], o_full[0][0][same])
    if device_rule:
        assert np.array_equal(npy(dst[3]).view(np.uint32), o_full[0][3].view(np.uint32))
    _rel(npy(d_eps), o[1])
    _rel(npy(d_L), o[2])
    for i in range(5):  # the log fields can sit near 0, where a relative tolerance alone is too strict
        np.testing.assert_allclose(npy(d_da)[:, i], o[3][i], rtol=1e-5, atol=1e-6)
    _rel(npy(d_st[0]), o[4][0])
    close(npy(d_st[1]), o[4][1])
    _rel(npy(d_count), rep)


def test_revert_keeps_the_whole_state():
    """handle_nans' revert: a chain whose output position is not finite keeps its whole state, random_generator_arg
    included, and its count still adds n; the others advance their key.  A Metropolis-adjusted transition rejects every
    proposal with a non-finite Delta, so the non-finite outputs are those of chains that start from one (q = inf)."""
    C, D = 64, 2
    tgt = T.UserTarget(2, plugin.read_example("bounded_gaussian"), np.array([5.0], F), name="bounded_gaussian",
                       dense_metric=False, general_integrators=True)
    rs = np.random.default_rng(3)
    q = tf(rs.uniform(-0.5, 0.5, (C, D)))
    st = amd.init(q, tgt, tk(oprng.key(5)))
    bad = torch.arange(C, device="cuda") % 3 == 0
    st.position[bad] = float("inf")
    eng = _engine.get_engine(st.position, tgt)
    eng.set_integrator(integrators.as_coefficients(TABLES["velocity_verlet"]))
    eng.ensure_metric(tf(np.ones(D, F)), diagonal_only=True)
    before = [t.clone() for t in st]
    state = [t.clone() for t in st]
    eps = tf(np.full(C, 1.0, F))
    L = tf(np.full(C, 3.0, F))
    da = tf(np.stack([np.full(C, x, F) for x in da_init(F(1.0))], 1))
    count = tf(np.zeros(C, F))
    ok, steps = ama.tune_step_(eng, tk(oprng.key(6)), state, eps, L, da, None, count, 1, True, 0.65,
                               device_rule=(_lib.AMCLMC_STEPS_RANDINT, 0))
    torch.cuda.synchronize()
    ok = ok.cpu()
    assert torch.equal(~ok, bad.cpu())
    badn = bad.cpu().numpy()
    for a, b in zip(state, before):
        assert np.array_equal(npy(a)[badn], npy(b)[badn])
    nxt = oprng.split(npy(before[3]).view(np.uint32), 2)[:, 1]
    assert np.array_equal(npy(state[3]).view(np.uint32)[ok.numpy()], nxt[ok.numpy()])
    assert np.array_equal(npy(count), npy(steps).astype(F)) and np.all(npy(steps) >= 1)


def _tune(tgt, st, key, kernel, num_steps=200, **kw):
    return bj.adjusted_mclmc_find_L_and_step_size(kernel, tgt, num_steps, st, key, 0.65, **kw)


def _uniform_kernel(**kw):
    return bj.adjusted_mclmc_dynamic.build_kernel(
        integration_steps_fn=amd.make_random_trajectory_length_fn(True, min_steps=0), **kw)


def test_native_tuner_bit_identity():
    D, C = 32, 96
    rs = np.random.default_rng(12)
    s = np.exp(rs.uniform(-1, 1, D))
    q0 = tf(rs.standard_normal((C, D)))
    key = tk(oprng.key(31))
    st = amd.init(q0, T.DiagGaussian(s), tk(oprng.key(32)))
    fin, par, n = _tune(T.DiagGaussian(s), st, key, _uniform_kernel(), frac_tune3=0.1)
    fin2, par2, n2 = _tune(T.DiagGaussian(s), st, key, _uniform_kernel(), frac_tune3=0.1, max_history_bytes=20 * D * 4 * 5)
    fin3, par3, n3 = _tune(_user_diag(s), st, key, _uniform_kernel(), frac_tune3=0.1)
    torch.cuda.synchronize()
    for other in ((fin2, par2, n2), (fin3, par3, n3)):
        for a, b in zip(list(fin) + list(par) + [n], list(other[0]) + list(other[1]) + [other[2]]):
            assert torch.equal(a, b)
    halves = []
    for lo in (0, C // 2):
        sub = bj.mcmc.dynamic_hmc.DynamicHMCState(*(t[lo:lo + C // 2].clone() for t in st))
        halves.append(_tune(T.DiagGaussian(s), sub, key, _uniform_kernel(chain_offset=lo), frac_tune3=0.1))
    torch.cuda.synchronize()
    for i in range(4):
        assert torch.equal(torch.cat([halves[0][0][i], halves[1][0][i]]), fin[i])
    for i in range(3):
        assert torch.equal(torch.cat([halves[0][1][i], halves[1][1][i]]), par[i])
    assert torch.equal(torch.cat([halves[0][2], halves[1][2]]), n)
    np.testing.assert_allclose(npy(par.L / par.step_size), 2.0, rtol=1e-6)


@pytest.mark.parametrize("frac_tune3, max_", [(0.0, "avg"), (0.1, "avg"), (0.1, "max")])
def test_native_tuner_matches_oracle(frac_tune3, max_):
    """A short tune (num_steps = 40: 4 + 4 steps in pass 1, 4 in pass 2, and with frac_tune3 = 0.1 four stage-3
    transitions, the ESS L update and another pass 1) with the randint rule, chain by chain against the oracle with
    per-chain keys.  Step counts and random_generator_arg are exact.  The parameters are held to 10 % and the final
    positions to 0.05: the dual averaging acts on acceptance rates exp(Delta) whose Delta is a small difference of
    log-densities, so the last-bit differences of those reductions move each step size by a little per step (up to 4 %
    seen), and the positions follow those step sizes (0.014 seen); a wrong key anywhere in the tree moves a position
    by O(1).  The teacher-forced tests pin the arithmetic itself."""
    D, C = 8, 5
    rs = np.random.default_rng(3)
    s = np.exp(rs.uniform(-1, 1, D))
    q0 = rs.standard_normal((C, D)).astype(F)
    keys = oprng.split(oprng.key(77), C)
    rga = oprng.split(oprng.key(78), C)
    st = amd.init(tf(q0), T.DiagGaussian(s), tk(rga))
    fin, par, n = _tune(T.DiagGaussian(s), st, tk(keys), bj.adjusted_mclmc_dynamic.build_kernel(), num_steps=40,
                        frac_tune3=frac_tune3, max=max_)
    ostate = tuple(npy(t) if i < 3 else rga for i, t in enumerate(st))
    ofin, (oL, oeps, oimm), on = at.find_L_and_step_size(("randint", 0), keys, 40, ostate, otargets.DiagGaussian(s),
                                                         TABLES["mclachlan"], 0.65, frac_tune3=frac_tune3, max_=max_)
    torch.cuda.synchronize()
    assert np.array_equal(npy(n), on.astype(np.int32))
    assert np.array_equal(npy(fin.random_generator_arg).view(np.uint32), ofin[3].view(np.uint32))
    np.testing.assert_allclose(npy(fin.position), ofin[0], rtol=0.05, atol=0.05)
    np.testing.assert_allclose(npy(par.step_size), oeps, rtol=0.1)
    np.testing.assert_allclose(npy(par.inverse_mass_matrix), oimm, rtol=0.1, atol=1e-4)
    np.testing.assert_allclose(npy(par.L), oL, rtol=0.1)


def test_fixed_rule_tune_advances_the_key_in_stage_3():
    """make_random_trajectory_length_fn(False): every tuning transition, stage 3's included, advances
    random_generator_arg, as the reference's kernel does; the final key is the oracle's."""
    D, C = 6, 4
    rs = np.random.default_rng(8)
    keys = oprng.split(oprng.key(80), C)
    rga = oprng.split(oprng.key(81), C)
    q0 = rs.standard_normal((C, D)).astype(F)
    st = amd.init(tf(q0), T.StdNormal(D), tk(rga))
    kernel = bj.adjusted_mclmc_dynamic.build_kernel(integration_steps_fn=amd.make_random_trajectory_length_fn(False))
    fin, par, n = _tune(T.StdNormal(D), st, tk(keys), kernel, num_steps=40, frac_tune3=0.1)
    ostate = tuple(npy(t) if i < 3 else rga for i, t in enumerate(st))
    ofin, _, on = at.find_L_and_step_size(("fixed", 1), keys, 40, ostate, otargets.DiagGaussian(np.ones(D)),
                                          TABLES["mclachlan"], 0.65, frac_tune3=0.1)
    torch.cuda.synchronize()
    assert np.array_equal(npy(fin.random_generator_arg).view(np.uint32), ofin[3].view(np.uint32))
    assert np.all(np.abs(npy(n) - on) <= 4)  # ceil(L / eps) may differ on a last-bit tie


@pytest.mark.parametrize("tk_", [2.0, 1.5])
def test_reference_ratio_on_every_chain(tk_):
    """test_tuner_returns_L_over_step_approx_target / _target_1p5 (:144-195) on 64 chains; then the median dynamic step
    count (:197-220) with target 2."""
    C, D = 64, 5
    rs = np.random.default_rng(int(tk_ * 10))
    st = amd.init(tf(rs.standard_normal((C, D))), T.StdNormal(D), tk(oprng.key(1)))
    _, par, _ = _tune(T.StdNormal(D), st, tk(oprng.key(2)), _uniform_kernel(), num_steps=4000,
                      target_num_integration_steps=tk_)
    np.testing.assert_allclose(npy(par.L / par.step_size), tk_, rtol=1e-5)
    if tk_ == 2.0:
        _, par_d, _ = bj.adjusted_mclmc_find_L_and_step_size(_uniform_kernel(), T.StdNormal(D), 4000, st, tk(oprng.key(3)),
                                                             0.65, frac_tune1=0.1, frac_tune2=0.1)
        np.testing.assert_allclose(npy(par_d.L / par_d.step_size), 2.0, rtol=1e-5)
        fn = amd.make_random_trajectory_length_fn(True, min_steps=0)
        _, _, acc, steps = bj.sample_adjusted_mclmc_native(
            tk(oprng.key(4)), st, T.StdNormal(D), par.step_size, 2000, integration_steps_fn=fn,
            integration_steps_params=(par.L / par.step_size,), inverse_mass_matrix=par.inverse_mass_matrix,
            keep_history=False)
        assert np.all(np.median(npy(steps).astype(F), axis=0) >= 1.5)


@pytest.mark.parametrize("dim, num_steps", [(10, 5000), (100, 8000), (300, 12000), (500, 16000)])
def test_high_dim_acceptance(dim, num_steps):
    """TestAdjustedMclmcHighDimAcceptance (:291-369) on 32 chains: L / step = 2, step > 0.01 sqrt(d), and a 200-step
    chain's mean acceptance within [0.45, 0.97]."""
    C = 32
    rs = np.random.default_rng(dim)
    st = amd.init(tf(rs.standard_normal((C, dim))), T.StdNormal(dim), tk(oprng.key(dim)))
    _, par, _ = _tune(T.StdNormal(dim), st, tk(oprng.key(dim + 1)), _uniform_kernel(), num_steps=num_steps)
    np.testing.assert_allclose(npy(par.L / par.step_size), 2.0, rtol=1e-5)
    assert np.all(npy(par.step_size) > 0.01 * math.sqrt(dim))
    fn = amd.make_random_trajectory_length_fn(True, min_steps=0)
    _, _, acc, _ = bj.sample_adjusted_mclmc_native(
        tk(oprng.key(dim + 2)), st, T.StdNormal(dim), par.step_size, 200, integration_steps_fn=fn,
        integration_steps_params=(par.L / par.step_size,), inverse_mass_matrix=par.inverse_mass_matrix,
        keep_history=False)
    a = npy(acc).mean(0)
    assert np.all((a >= 0.45) & (a <= 0.97)), a


def _regression():
    rs = np.random.default_rng(42)
    x = rs.standard_normal((1000, 1)).astype(F)
    y = (3 * x[:, 0] + rs.standard_normal(1000)).astype(F)
    return T.LinearRegression(x, y)


@pytest.mark.parametrize("dynamic", [True, False])
def test_regression_posterior_with_the_tuner(dynamic):
    """test_sampling.py:432-480 with the tuner (frac_tune3 = 0.1), static (target 0.9) and dynamic (target 0.65): on every
    chain the mean scale is 1 +- 0.1 and the mean coefficient 3 +- 0.1 after 3000 burn-in steps.  Positions are
    (log_scale, coefs) as in the MCLMC tuner's regression test."""
    tgt = _regression()
    C = 32
    q0 = tf(np.ones((C, 2)))
    if dynamic:
        st = amd.init(q0, tgt, tk(oprng.key(7)))
        kernel, target = _uniform_kernel(), 0.65
    else:
        st = bj.adjusted_mclmc.init(q0, tgt)
        kernel, target = bj.adjusted_mclmc.build_kernel(), 0.9
    fin, par, _ = bj.adjusted_mclmc_find_L_and_step_size(kernel, tgt, 10000, st, tk(oprng.key(8)), target, frac_tune3=0.1,
                                                         diagonal_preconditioning=False)
    avg = par.L / par.step_size
    if dynamic:
        _, hist, _, _ = bj.sample_adjusted_mclmc_native(
            tk(oprng.key(9)), fin, tgt, par.step_size, 10000,
            integration_steps_fn=amd.make_random_trajectory_length_fn(True, min_steps=0), integration_steps_params=(avg,),
            inverse_mass_matrix=par.inverse_mass_matrix)
    else:
        _, hist, _, _ = bj.sample_adjusted_mclmc_native(tk(oprng.key(9)), fin, tgt, par.step_size, 10000,
                                                        num_integration_steps=avg,
                                                        inverse_mass_matrix=par.inverse_mass_matrix)
    h = npy(hist)[3000:]
    assert np.all(np.abs(np.exp(h[..., 0]).mean(0) - 1.0) < 0.1)
    assert np.all(np.abs(h[..., 1].mean(0) - 3.0) < 0.1)


@pytest.mark.parametrize("rule", ["static", "uniform", "fixed"])
def test_tuned_parameters_feed_the_samplers(rule):
    """Per-chain L / step_size in the step API and the native loop: the same draws, and the step counts of the rule."""
    C, D, T_ = 16, 6, 5
    rs = np.random.default_rng(5)
    tgt = T.DiagGaussian(np.linspace(0.5, 2, D))
    eps = tf(rs.uniform(0.3, 0.8, C))
    avg = tf(rs.uniform(1.2, 4.5, C))
    key = tk(oprng.key(11))
    q0 = tf(rs.standard_normal((C, D)))
    if rule == "static":
        st = bj.adjusted_mclmc.init(q0, tgt)
        alg = bj.adjusted_mclmc(tgt, eps, num_integration_steps=avg)
        fin, hist, _, steps = bj.sample_adjusted_mclmc_native(key, st, tgt, eps, T_, num_integration_steps=avg)
        want = np.ceil(npy(avg)).astype(np.int32)
    else:
        fn = amd.make_random_trajectory_length_fn(rule == "uniform", min_steps=0 if rule == "uniform" else 1)
        st = amd.init(q0, tgt, tk(oprng.key(12)))
        alg = bj.adjusted_mclmc_dynamic(tgt, eps, integration_steps_fn=fn, integration_steps_params=(avg,))
        fin, hist, _, steps = bj.sample_adjusted_mclmc_native(key, st, tgt, eps, T_, integration_steps_fn=fn,
                                                              integration_steps_params=(avg,))
        if rule == "uniform":
            rgas, r = [], npy(st.random_generator_arg).view(np.uint32)
            for _ in range(T_):
                rgas.append(r)
                r = oprng.split(r, 2)[:, 1]
            want = np.stack([np.maximum(np.ceil((oprng.uniform(r) * np.array([ao.rescale(a) for a in npy(avg)], F))
                                                .astype(F)), 0) for r in rgas]).astype(np.int32)
        else:
            want = np.maximum(np.ceil(npy(avg)), 1).astype(np.int32)
    keys = bj.random.split(key, T_)
    state = st
    for t in range(T_):
        state, info = alg.step(keys[t], state)
        assert torch.equal(state.position, hist[t])
    assert torch.equal(state.position, fin.position)
    if rule != "static":
        assert torch.equal(state.random_generator_arg, fin.random_generator_arg)
    s = npy(steps)
    assert np.array_equal(s, np.broadcast_to(want, s.shape))


def test_rejections():
    rs = np.random.default_rng(0)
    key = tk(oprng.key(0))
    kernel = bj.adjusted_mclmc.build_kernel()
    for D in (1, 1028):
        q = tf(rs.standard_normal((8, D)))
        st = bj.mcmc.hmc.HMCState(q, tf(np.zeros(8)), q.clone())
        with pytest.raises(_lib.BjxError, match="error -2"):
            bj.adjusted_mclmc_find_L_and_step_size(kernel, T.StdNormal(D), 100, st, key, 0.9)
    tgt = T.DenseGaussian(np.eye(132, dtype=F))
    q = tf(rs.standard_normal((8, 132)))
    st = bj.mcmc.hmc.HMCState(q, tf(np.zeros(8)), q.clone())
    with pytest.raises(_lib.BjxError, match="error -2"):
        bj.adjusted_mclmc_find_L_and_step_size(kernel, tgt, 100, st, key, 0.9)
    from blackjax_b200.mcmc.metrics import LowRankMetric
    D = 64
    q = tf(rs.standard_normal((8, D)))
    st = [q, tf(np.zeros(8)), q.clone()]
    for imm in (tf(np.broadcast_to(np.eye(D, dtype=F), (8, D, D))),
                LowRankMetric(torch.ones(D), torch.eye(D, 2), torch.full((2,), 2.0))):
        eng = _engine.get_engine(q, T.StdNormal(D))
        eng.ensure_metric(imm)
        with pytest.raises(_lib.BjxError, match="error -2"):
            ama.tune_step_(eng, key, st, torch.ones(8, device="cuda"), torch.full((8,), 2.0, device="cuda"),
                           torch.zeros(8, 5, device="cuda"), None, None, 1, True, 0.9)
    hst = bj.mcmc.hmc.HMCState(*st)
    with pytest.raises(TypeError):
        bj.adjusted_mclmc_find_L_and_step_size(bj.hmc.build_kernel(), T.StdNormal(D), 100, hst, key, 0.9)
    with pytest.raises(ValueError):
        bj.adjusted_mclmc_find_L_and_step_size(
            bj.adjusted_mclmc_dynamic.build_kernel(integration_steps_fn=lambda k, a: 3), T.StdNormal(D), 100,
            amd.init(q, T.StdNormal(D), key), key, 0.9)
    with pytest.raises(ValueError):
        bj.adjusted_mclmc_find_L_and_step_size(kernel, T.StdNormal(D), 10, hst, key, 0.9, frac_tune3=0.1)
