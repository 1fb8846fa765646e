"""Adjusted MCLMC / MAMS on the GPU (k_amclmc_transition through bjx_adjusted_mclmc_step / bjx_adjusted_mclmc_sample)
against the float32 restatement in oracle/adjusted_mclmc.py on the same state and keys.

* one transition, teacher-forced: the proposal (q, unit momentum), the drawn momentum, energy, and the new q, logp, grad
  within 1e-5 relative (close() of test_gpu_parity), p_accept within 1e-5 of the log-density scale, and accept decisions
  identical except where the uniform lies within that tolerance of p_accept.
  Every warp size class, every built-in row target, a plug-in, all four tables, finite and infinite L_proposal_factor,
  scalar and per-chain step size, per-chain step counts including 0 and 1, [D] and [C, D] metrics;
* the plug-in diagonal Gaussian is bit-identical to the built-in target;
* bjx_adjusted_mclmc_sample is bit-identical to T step calls for the static sampler and both device step rules (with the
  advanced random_generator_arg), and two handles of C/2 chains with chain_offset to one handle of C;
* configurations that are not built are rejected with BJX_E_UNSUPPORTED;
* the Metropolis correction: per-dimension mean and variance of a spread diagonal Gaussian within a z-bound, MCSE from the
  device ESS, at a step size where unadjusted MCLMC is visibly biased (tests/test_adjusted_mclmc_oracle.py);
* the reference's regression posterior (tests/mcmc/test_sampling.py:432-480), static and dynamic.
"""
import math

import numpy as np
import pytest
import torch

import blackjax_b200 as bj
from blackjax_b200 import _lib, plugin, targets as T
from blackjax_b200.mcmc import adjusted_mclmc_dynamic as amd
from blackjax_b200.mcmc import integrators
from oracle import adjusted_mclmc as oa
from oracle import prng as oprng
from oracle import targets as otargets
from test_gpu_parity import close, npy, tf, tk

pytestmark = pytest.mark.gpu
F = np.float32
TABLES = {"velocity_verlet": integrators.isokinetic_velocity_verlet, "mclachlan": integrators.isokinetic_mclachlan,
          "yoshida": integrators.isokinetic_yoshida, "omelyan": integrators.isokinetic_omelyan}


def _user_diag(s):
    inv_var = (1.0 / (np.asarray(s, np.float64) ** 2)).astype(F)
    return T.UserTarget(len(s), plugin.read_example("diag_gaussian"), inv_var, name="diag_gaussian")


def _targets(name, D, rs):
    """(device target, oracle target, initial position scale)"""
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


CASES = (
    # (target, D, table, metric, L_proposal_factor, per-chain step size)
    [("diag", D, "mclachlan", "shared", 1.0, False) for D in (2, 18, 70, 100, 128, 256, 512, 1024)]
    + [("diag", 100, t, "shared", 1.0, False) for t in ("velocity_verlet", "yoshida", "omelyan")]
    + [("diag", 256, "mclachlan", "per_chain", 1.0, True), ("diag", 70, "velocity_verlet", "per_chain", math.inf, False),
       ("diag", 512, "omelyan", "shared", math.inf, True), ("diag", 1024, "velocity_verlet", "per_chain", 0.7, True),
       ("funnel", 100, "mclachlan", "shared", 1.0, False), ("funnel", 256, "velocity_verlet", "per_chain", math.inf, True),
       ("banana", 2, "mclachlan", "shared", 1.0, False), ("banana", 2, "yoshida", "per_chain", math.inf, True),
       ("dense", 64, "mclachlan", "shared", 1.0, False), ("dense", 128, "omelyan", "per_chain", 2.0, True),
       ("dense", 30, "velocity_verlet", "shared", math.inf, False),
       ("user_diag", 100, "mclachlan", "per_chain", 1.0, True), ("user_diag", 100, "velocity_verlet", "shared", math.inf,
                                                                   False)])


@pytest.mark.parametrize("name, D, table, metric, L_factor, per_chain", CASES)
def test_transition_matches_oracle(name, D, table, metric, L_factor, per_chain):
    rs = np.random.default_rng(D * 11 + len(name) + len(table))
    C = 67
    tgt, otgt, scale = _targets(name, D, rs)
    q = (scale * rs.standard_normal((C, D))).astype(F)
    logp, g = otgt(q)
    imm = np.exp(rs.uniform(-0.5, 0.5, (C, D) if metric == "per_chain" else D)).astype(F)
    base_eps = 0.2 * math.sqrt(D) if name != "funnel" else 0.03 * math.sqrt(D)
    eps = (base_eps * rs.uniform(0.5, 1.5, C)).astype(F) if per_chain else F(base_eps)
    n = rs.integers(0, 5, C).astype(np.int32)
    n[:3] = (0, 1, 4)
    step_key = oprng.key(2000 + D)
    keys = oprng.split(step_key, C)  # chain c of a shared step key uses split(step_key, C)[c]
    (oq, ologp, og), oinfo = oa.adjusted_mclmc_kernel(keys, (q, logp, g), otgt, imm, eps, n, TABLES[table], L_factor)

    st = bj.mcmc.hmc.HMCState(tf(q), tf(logp), tf(g))
    eps_arg = tf(eps) if per_chain else float(eps)
    kernel = bj.adjusted_mclmc.build_kernel(integrator=TABLES[table], full_info=True)
    new, info = kernel(tk(step_key), st, tgt, eps_arg, (torch.from_numpy(n).cuda(),), tf(imm), L_factor)
    torch.cuda.synchronize()
    lscale = max(float(np.max(np.abs(logp))), 1.0)
    close(npy(info.momentum), oinfo.momentum, scale=1.0 / math.sqrt(D))
    close(npy(info.proposal.position), oinfo.proposal[0])
    close(npy(info.proposal.momentum), oinfo.proposal[1], scale=1.0 / math.sqrt(D))
    close(npy(info.energy), oinfo.energy, scale=lscale)
    # p_accept = min(1, exp(Delta)) and Delta is a difference of log-densities, accurate to 1e-5 of their scale: so is
    # p_accept, and decisions may differ only where the uniform lies that close to it
    close(npy(info.acceptance_rate), oinfo.acceptance_rate, scale=lscale)
    acc = npy(info.is_accepted)
    tie = np.abs(oinfo.uniform.astype(np.float64) - oinfo.acceptance_rate) < 1e-5 * lscale
    assert np.array_equal(acc[~tie], oinfo.is_accepted[~tie])
    assert np.all(acc[n == 0]) and np.all(npy(info.acceptance_rate)[n == 0] == 1)
    assert np.array_equal(npy(info.is_divergent)[~tie], oinfo.is_divergent[~tie])
    same = acc == oinfo.is_accepted
    assert same.mean() > 0.9
    close(npy(new.position)[same], oq[same])
    close(npy(new.logdensity_grad)[same], og[same])
    close(npy(new.logdensity)[same], ologp[same], scale=lscale)
    rej = ~acc
    assert np.array_equal(npy(new.position)[rej], q[rej]) and np.array_equal(npy(new.logdensity)[rej], logp[rej])
    np.testing.assert_allclose(np.linalg.norm(npy(info.proposal.momentum), axis=1), 1.0, rtol=2e-6)


def test_in_place_rejection_writes_nothing_and_out_of_place_copies():
    D, C = 64, 256
    rs = np.random.default_rng(1)
    tgt = T.DiagGaussian(np.exp(rs.uniform(-1, 1, D)))
    st = bj.adjusted_mclmc.init(tf(rs.standard_normal((C, D))), tgt)
    key = tk(oprng.key(3))
    out, info = bj.adjusted_mclmc.build_kernel()(key, st, tgt, 3.0, (6,), 1.0, 1.0)
    st2 = bj.mcmc.hmc.HMCState(*(t.clone() for t in st))
    ref = bj.mcmc.hmc.HMCState(*(t.clone() for t in st))
    inp, info2 = bj.adjusted_mclmc.build_kernel(inplace=True)(key, st2, tgt, 3.0, (6,), 1.0, 1.0)
    torch.cuda.synchronize()
    acc = npy(info.is_accepted)
    assert 0 < acc.mean() < 1
    for a, b in zip(out, inp):
        assert torch.equal(a, b)
    assert inp.position.data_ptr() == st2.position.data_ptr()
    for a, b in zip(out, ref):
        assert torch.equal(a[torch.from_numpy(~acc).cuda()], b[torch.from_numpy(~acc).cuda()])


def test_plugin_bit_identical_to_builtin():
    D, C = 100, 67
    rs = np.random.default_rng(5)
    s = np.exp(rs.uniform(-1, 1, D))
    imm = tf(np.exp(rs.uniform(-0.5, 0.5, D)))
    q = tf(rs.standard_normal((C, D)))
    key = tk(oprng.key(11))
    n = torch.from_numpy(rs.integers(0, 7, C).astype(np.int32)).cuda()
    out = []
    for tgt in (T.DiagGaussian(s), _user_diag(s)):
        st = bj.adjusted_mclmc.init(q, tgt)
        new, info = bj.adjusted_mclmc.build_kernel(full_info=True)(key, st, tgt, 2.5, (n,), imm, 1.3)
        out.append([*st, *new, info.energy, info.acceptance_rate, info.proposal.position, info.proposal.momentum])
    torch.cuda.synchronize()
    for a, b in zip(*out):
        assert torch.equal(a, b)


def _loop_problem(C=96, D=128):
    rs = np.random.default_rng(9)
    tgt = T.DiagGaussian(np.exp(rs.uniform(-1, 1, D)))
    imm = tf(np.exp(rs.uniform(-0.5, 0.5, D)))
    q0 = tf(rs.standard_normal((C, D)))
    eps = tf(rs.uniform(1.0, 3.0, C))
    return tgt, imm, q0, eps


def test_native_loop_static_bit_identical():
    tgt, imm, q0, eps = _loop_problem()
    C, Tn = q0.shape[0], 20
    key = tk(oprng.key(21))
    st = bj.adjusted_mclmc.init(q0, tgt)
    fin, hist, acc, steps = bj.sample_adjusted_mclmc_native(key, st, tgt, eps, Tn, num_integration_steps=5,
                                                             L_proposal_factor=1.2, inverse_mass_matrix=imm, thin=4)
    kernel = bj.adjusted_mclmc.build_kernel()
    step_keys = bj.random.split(key, Tn)
    s, rows, accs = st, [], []
    for t in range(Tn):
        s, info = kernel(step_keys[t], s, tgt, eps, (5,), imm, 1.2)
        accs.append(info.acceptance_rate)
        if (t + 1) % 4 == 0:
            rows.append(s.position)
    torch.cuda.synchronize()
    for a, b in zip(fin, s):
        assert torch.equal(a, b)
    assert torch.equal(hist, torch.stack(rows)) and torch.equal(acc, torch.stack(accs))
    assert bool((steps == 5).all())
    assert 0.2 < float(acc.mean()) < 1.0
    halves = []
    for lo in (0, C // 2):
        sub = bj.mcmc.hmc.HMCState(*(t[lo:lo + C // 2].clone() for t in st))
        f, _, _, _ = bj.sample_adjusted_mclmc_native(key, sub, tgt, eps[lo:lo + C // 2].contiguous(), Tn,
                                                     num_integration_steps=5, L_proposal_factor=1.2,
                                                     inverse_mass_matrix=imm, keep_history=False, chain_offset=lo)
        halves.append(f)
    torch.cuda.synchronize()
    for i in range(3):
        assert torch.equal(torch.cat([halves[0][i], halves[1][i]]), fin[i])


@pytest.mark.parametrize("rule", ["randint", "uniform", "uniform_unclipped"])
def test_native_loop_dynamic_bit_identical(rule):
    tgt, imm, q0, eps = _loop_problem()
    C, Tn, avg = q0.shape[0], 16, 4.6
    key = tk(oprng.key(31))
    if rule == "randint":
        fn, params, ofn = amd._integration_steps, (), oa.steps_randint
    else:
        m = 0 if rule == "uniform_unclipped" else 1
        fn, params = amd.make_random_trajectory_length_fn(True, min_steps=m), (avg,)
        ofn = lambda k: oa.steps_uniform(k, avg, m)  # noqa: E731
    rga0 = oprng.split(oprng.key(77), C)
    st = bj.adjusted_mclmc_dynamic.init(q0, tgt, tk(rga0))
    fin, hist, acc, steps = bj.sample_adjusted_mclmc_native(key, st, tgt, eps, Tn, integration_steps_fn=fn,
                                                             integration_steps_params=params, L_proposal_factor=1.0,
                                                             inverse_mass_matrix=imm)
    kernel = bj.adjusted_mclmc_dynamic.build_kernel(integration_steps_fn=fn)
    step_keys = bj.random.split(key, Tn)
    s, rows, accs, ns = st, [], [], []
    for t in range(Tn):
        n_t = fn(s.random_generator_arg, *params)
        s, info = kernel(step_keys[t], s, tgt, eps, 1.0, imm, params)
        rows.append(s.position)
        accs.append(info.acceptance_rate)
        ns.append(n_t)
    torch.cuda.synchronize()
    for a, b in zip(fin, s):
        assert torch.equal(a, b)
    assert torch.equal(hist, torch.stack(rows)) and torch.equal(acc, torch.stack(accs))
    assert torch.equal(steps, torch.stack(ns).to(torch.int32))
    # the step counts and the advanced random_generator_arg are the reference's rule and split(key)[1]
    rga, on = rga0, []
    for t in range(Tn):
        on.append(ofn(rga))
        rga = oprng.split(rga, 2)[:, 1]
    assert np.array_equal(npy(steps), np.stack(on))
    assert np.array_equal(npy(fin.random_generator_arg.view(torch.int32)).view(np.uint32), rga)


def test_unsupported_configurations_are_rejected():
    rs = np.random.default_rng(0)
    key = tk(oprng.key(0))

    def step(tgt, D, imm, C=8):
        st = bj.adjusted_mclmc.init(tf(rs.standard_normal((C, D))), tgt)
        return bj.adjusted_mclmc.build_kernel()(key, st, tgt, 0.5, (3,), imm)

    from blackjax_b200.mcmc.metrics import LowRankMetric
    for D, imm in ((8, None), (64, "dense3"), (64, "low_rank"), (1028, 1.0)):
        tgt = T.StdNormal(D)
        if imm is None:  # a dense Gaussian target beyond 128 dims
            tgt, imm = T.DenseGaussian(np.eye(132, dtype=F)), 1.0
            D = 132
        elif imm == "dense3":
            imm = tf(np.broadcast_to(np.eye(D, dtype=F), (8, D, D)))
        elif imm == "low_rank":
            imm = LowRankMetric(torch.ones(D), torch.eye(D, 2), torch.full((2,), 2.0))
        with pytest.raises(_lib.BjxError, match="error -2: adjusted MCLMC"):
            step(tgt, D, imm)
    with pytest.raises(_lib.BjxError, match="error -2: adjusted MCLMC needs dim >= 2"):
        step(T.StdNormal(1), 1, 1.0)


def _ess(hist, tgt):
    return npy(bj.diagnostics.effective_sample_size(hist.contiguous(), tgt))


def test_metropolis_correction_recovers_gaussian_moments():
    """A diagonal Gaussian with scales 0.5 .. 4 and its own metric, L_proposal_factor = 1, 4 steps of 4.0 per transition
    (mean acceptance about 0.67; unadjusted MCLMC at this step size underestimates the variance by about 12 %, see
    tests/test_adjusted_mclmc_oracle.py).  Per-dimension mean and variance within 5 MCSE of the truth, the MCSE from the
    device ESS of x and of x^2."""
    scales = np.array([0.5, 1.0, 2.0, 4.0])
    D, C, Tn = 4, 4096, 400
    tgt = T.DiagGaussian(scales)
    rs = np.random.default_rng(3)
    st = bj.adjusted_mclmc.init(tf(scales * rs.standard_normal((C, D))), tgt)
    _, hist, acc, _ = bj.sample_adjusted_mclmc_native(tk(oprng.key(5)), st, tgt, 4.0, Tn, num_integration_steps=4,
                                                       L_proposal_factor=1.0, inverse_mass_matrix=tf(scales ** 2))
    assert 0.6 < float(acc[50:].mean()) < 0.8
    x = hist[50:] / tf(scales)
    xn = npy(x).reshape(-1, D)
    n_mean = _ess(x, tgt)
    sq = (x * x).contiguous()
    n_var = _ess(sq, tgt)
    z_mean = np.abs(xn.mean(0)) / (xn.std(0) / np.sqrt(n_mean))
    z_var = np.abs((xn * xn).mean(0) - 1.0) / ((xn * xn).std(0) / np.sqrt(n_var))
    assert np.all(z_mean < 5), (z_mean, n_mean)
    assert np.all(z_var < 5), (z_var, n_var, (xn * xn).mean(0))


def _regression():
    rs = np.random.default_rng(42)
    x = rs.standard_normal((1000, 1)).astype(F)
    y = (3 * x[:, 0] + rs.standard_normal(1000)).astype(F)
    return T.LinearRegression(x, y)


@pytest.mark.parametrize("dynamic", [False, True])
def test_regression_posterior(dynamic):
    """tests/mcmc/test_sampling.py:432-480 with fixed parameters in place of the tuner: step size 0.8 in the frame of the
    metric diag(0.03^2, 0.03^2), L_proposal_factor = inf, mean 4 steps (static: 4; dynamic: ceil(U rescale(4))); 512 chains
    from (log_scale, coefs) = (1, 1), 1000 transitions, the first 300 dropped: mean scale 1 +- 0.1 and mean coefficient
    3 +- 0.1."""
    tgt = _regression()
    C, Tn = 512, 1000
    q0 = tf(np.ones((C, 2)))
    imm = tf(np.array([0.03 ** 2, 0.03 ** 2]))
    key = tk(oprng.key(8))
    if dynamic:
        st = bj.adjusted_mclmc_dynamic.init(q0, tgt, tk(oprng.key(9)))
        kw = dict(integration_steps_fn=amd.make_random_trajectory_length_fn(True, min_steps=0),
                  integration_steps_params=(4.0,))
    else:
        st = bj.adjusted_mclmc.init(q0, tgt)
        kw = dict(num_integration_steps=4)
    _, hist, acc, _ = bj.sample_adjusted_mclmc_native(key, st, tgt, 0.8, Tn, inverse_mass_matrix=imm, **kw)
    h = npy(hist[300:])
    assert float(acc[300:].mean()) > 0.3
    np.testing.assert_allclose(np.mean(np.exp(h[..., 0])), 1.0, rtol=1e-2, atol=1e-1)
    np.testing.assert_allclose(np.mean(h[..., 1]), 3.0, rtol=1e-2, atol=1e-1)


def test_dynamic_top_level_api_runs_many_chains():
    """blackjax.adjusted_mclmc_dynamic(target, step_size=..., inverse_mass_matrix=...) -> init / step over 65536 chains."""
    D, C = 16, 65536
    tgt = T.DiagGaussian(np.linspace(0.5, 2.0, D))
    alg = bj.adjusted_mclmc_dynamic(tgt, step_size=1.0, inverse_mass_matrix=tf(np.linspace(0.5, 2.0, D) ** 2))
    st = alg.init(tf(np.random.default_rng(0).standard_normal((C, D))), tk(oprng.key(1)))
    assert tuple(st.random_generator_arg.shape) == (C, 2)
    st2, info = alg.step(tk(oprng.key(2)), st)
    torch.cuda.synchronize()
    assert st2.position.shape == (C, D) and info.acceptance_rate.shape == (C,)
    assert 0.3 < float(info.acceptance_rate.mean()) <= 1.0
    n = npy(info.num_integration_steps)
    assert n.min() >= 1 and n.max() <= 9
