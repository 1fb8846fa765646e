"""MCLMC on the GPU (k_mclmc_transition through bjx_mclmc_init / bjx_mclmc_step / bjx_mclmc_sample) against the float32
restatement in oracle/mclmc.py on the same state and keys.

* init: the momentum is the oracle's unit vector within 1e-6;
* one transition, teacher-forced: q, p, logp, grad and the energy change within 1e-5 relative (close(): abs floor 5 % of the
  row maximum for q and grad, 1/sqrt(D) -- the RMS component of a unit vector -- for p, the log-density scale for the
  reductions), nonans identical; every warp size class, every
  built-in row target, a plug-in, shared and per-chain metrics, all four tables, finite and infinite L, scalar and
  per-chain step size and L;
* the plug-in diagonal Gaussian is bit-identical to the built-in target;
* bjx_mclmc_sample is bit-identical to T calls of bjx_mclmc_step, and two handles of C/2 chains with chain_offset to one
  handle of C;
* the reference's NaN cases (#969) on its bounded target revert to finite states with nonans = False;
* a finite energy cutoff reverts exactly the chains the oracle reverts (handle_high_energy on the device);
* configurations that are not built are rejected with BJX_E_UNSUPPORTED;
* a long run on a scaled Gaussian recovers its mean and variance.
"""
import math

import numpy as np
import pytest
import torch

import blackjax_b200 as bj
from blackjax_b200 import _lib, plugin, targets as T
from blackjax_b200.mcmc import integrators
from oracle import mclmc as om
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


def _state(D, C, otgt, scale, rs):
    q = (scale * rs.standard_normal((C, D))).astype(F)
    u = rs.standard_normal((C, D))
    u = (u / np.linalg.norm(u, axis=1, keepdims=True)).astype(F)
    logp, g = otgt(q)
    return q, u, logp, g


CASES = (
    # (target, D, table, metric, L, per_chain)
    [("diag", D, "mclachlan", "shared", "finite", False) for D in (2, 18, 70, 100, 128, 256, 512, 1024)]
    + [("diag", 100, t, "shared", "finite", False) for t in ("velocity_verlet", "yoshida", "omelyan")]
    + [("diag", 256, "mclachlan", "per_chain", "finite", True), ("diag", 70, "velocity_verlet", "per_chain", "inf", False),
       ("diag", 512, "omelyan", "shared", "inf", True), ("diag", 1024, "velocity_verlet", "per_chain", "finite", True),
       ("funnel", 100, "mclachlan", "shared", "finite", False), ("funnel", 256, "velocity_verlet", "per_chain", "finite", True),
       ("banana", 2, "mclachlan", "shared", "finite", False), ("banana", 2, "yoshida", "per_chain", "inf", True),
       ("dense", 64, "mclachlan", "shared", "finite", False), ("dense", 128, "omelyan", "per_chain", "finite", True),
       ("dense", 30, "velocity_verlet", "shared", "inf", False),
       ("user_diag", 100, "mclachlan", "per_chain", "finite", True), ("user_diag", 100, "velocity_verlet", "shared", "inf",
                                                                       False)])


@pytest.mark.parametrize("name, D, table, metric, Lkind, per_chain", CASES)
def test_transition_matches_oracle(name, D, table, metric, Lkind, per_chain):
    rs = np.random.default_rng(D * 7 + len(name) + len(table))
    C = 67
    tgt, otgt, scale = _targets(name, D, rs)
    q, u, logp, g = _state(D, C, otgt, scale, rs)
    imm = np.exp(rs.uniform(-0.5, 0.5, (C, D) if metric == "per_chain" else D)).astype(F)
    base_eps = 0.3 * math.sqrt(D) if name != "funnel" else 0.05 * math.sqrt(D)
    if per_chain:
        eps = (base_eps * rs.uniform(0.5, 1.5, C)).astype(F)
        L = (math.sqrt(D) * rs.uniform(0.5, 2.0, C)).astype(F) if Lkind == "finite" else np.full(C, np.inf, F)
    else:
        eps = F(base_eps)
        L = F(math.sqrt(D)) if Lkind == "finite" else F(np.inf)
    step_key = oprng.key(1000 + D)
    keys = oprng.split(step_key, C)  # chain c of a shared step key uses split(step_key, C)[c]
    (oq, ou, ologp, og), oinfo = om.mclmc_kernel(keys, (q, u, logp, g), otgt, imm, L, eps, TABLES[table])

    st = bj.mcmc.hmc.IntegratorState(tf(q), tf(u), tf(logp), tf(g))
    as_dev = (lambda x: tf(x)) if per_chain else float
    new, info = bj.mclmc.build_kernel(integrator=TABLES[table])(tk(step_key), st, tgt, tf(imm), as_dev(L), as_dev(eps))
    torch.cuda.synchronize()
    assert np.array_equal(npy(info.nonans), oinfo.nonans)
    close(npy(new.position), oq)
    close(npy(new.momentum), ou, scale=1.0 / math.sqrt(D))  # a unit vector: floor = its RMS component
    close(npy(new.logdensity_grad), og)
    lscale = max(float(np.max(np.abs(logp))), 1.0)
    close(npy(new.logdensity), ologp, scale=lscale)
    close(npy(info.energy_change), oinfo.energy_change, scale=lscale)
    close(npy(info.kinetic_change), oinfo.kinetic_change, scale=lscale)
    np.testing.assert_allclose(np.linalg.norm(npy(new.momentum), axis=1), 1.0, rtol=2e-6)


@pytest.mark.parametrize("D", [18, 256])
def test_high_energy_cutoff_matches_oracle(D):
    """handle_high_energy on the device (mclmc.py:257-281): a finite cutoff between the chains' |energy_change| values
    reverts the chains above it (previous q, logp, grad; unit momentum from the cutoff key; zero energy and kinetic
    change) and lets the others through, as the oracle does."""
    rs = np.random.default_rng(40 + D)
    C = 67
    tgt, otgt, _ = _targets("diag", D, rs)
    q, u, logp, g = _state(D, C, otgt, 1.0, rs)
    imm = np.exp(rs.uniform(-0.5, 0.5, D)).astype(F)
    eps, L = F(0.6 * math.sqrt(D)), F(math.sqrt(D))
    step_key = oprng.key(77 + D)
    keys = oprng.split(step_key, C)
    table = TABLES["mclachlan"]
    _, free = om.mclmc_kernel(keys, (q, u, logp, g), otgt, imm, L, eps, table)
    e = np.sort(np.abs(free.energy_change.astype(np.float64)))
    mid = C // 2
    cutoff = 0.5 * (e[mid - 1] + e[mid])
    var = 5e-4
    ratio = cutoff * cutoff / (D * var)
    cut32 = bj.mcmc.mclmc.energy_cutoff(D, ratio, var)  # the float32 value the kernel receives
    (oq, ou, ologp, og), oinfo = om.mclmc_kernel(keys, (q, u, logp, g), otgt, imm, L, eps, table, cutoff=cut32)
    high = np.abs(free.energy_change) > F(cut32)
    assert 0 < high.sum() < C
    st = bj.mcmc.hmc.IntegratorState(tf(q), tf(u), tf(logp), tf(g))
    new, info = bj.mclmc.build_kernel(integrator=table, desired_energy_var_max_ratio=ratio, desired_energy_var=var)(
        tk(step_key), st, tgt, tf(imm), float(L), float(eps))
    torch.cuda.synchronize()
    assert np.array_equal(npy(info.nonans), oinfo.nonans) and oinfo.nonans.all()
    pos, mom, lp, gr = (npy(t) for t in new)
    assert np.array_equal(pos[high], q[high]) and np.array_equal(gr[high], g[high]) and np.array_equal(lp[high], logp[high])
    assert np.all(npy(info.energy_change)[high] == 0) and np.all(npy(info.kinetic_change)[high] == 0)
    np.testing.assert_allclose(mom[high], ou[high], rtol=0, atol=1e-6)
    assert not np.array_equal(pos[~high], q[~high])
    close(pos, oq)
    close(mom, ou, scale=1.0 / math.sqrt(D))
    close(gr, og)
    lscale = max(float(np.max(np.abs(logp))), 1.0)
    close(lp, ologp, scale=lscale)
    close(npy(info.energy_change), oinfo.energy_change, scale=lscale)


@pytest.mark.parametrize("D", [2, 100, 1024])
def test_init_unit_vector(D):
    rs = np.random.default_rng(D)
    C = 45
    q = rs.standard_normal((C, D)).astype(F)
    keys = oprng.split(oprng.key(D), C)
    st = bj.mclmc.init(tf(q), T.StdNormal(D), tk(keys))
    oq, ou, ologp, og = om.mclmc_init(q, otargets.StdNormal(D), keys)
    torch.cuda.synchronize()
    np.testing.assert_allclose(npy(st.momentum), ou, rtol=0, atol=1e-6)
    close(npy(st.logdensity_grad), og)
    close(npy(st.logdensity), ologp, scale=float(np.max(np.abs(ologp))))


def test_plugin_bit_identical_to_builtin():
    D, C = 100, 67
    rs = np.random.default_rng(5)
    s = np.exp(rs.uniform(-1, 1, D))
    imm = tf(np.exp(rs.uniform(-0.5, 0.5, D)))
    q = tf(rs.standard_normal((C, D)))
    key = tk(oprng.key(11))
    out = []
    for tgt in (T.DiagGaussian(s), _user_diag(s)):
        st = bj.mclmc.init(q, tgt, key)
        new, info = bj.mclmc.build_kernel()(key, st, tgt, imm, 7.0, 2.5)
        out.append([*st, *new, info.energy_change, info.kinetic_change])
    torch.cuda.synchronize()
    for a, b in zip(*out):
        assert torch.equal(a, b)


def test_native_loop_and_chain_offset_bit_identical():
    D, C, Tn = 128, 96, 24
    rs = np.random.default_rng(9)
    tgt = T.DiagGaussian(np.exp(rs.uniform(-1, 1, D)))
    imm = tf(np.exp(rs.uniform(-0.5, 0.5, D)))
    q0 = tf(rs.standard_normal((C, D)))
    eps, L = tf(rs.uniform(1.0, 3.0, C)), 9.0
    key = tk(oprng.key(21))
    st = bj.mclmc.init(q0, tgt, key)
    fin, hist, de = bj.sample_mclmc_native(key, st, tgt, L, eps, Tn, inverse_mass_matrix=imm, thin=3)
    kernel = bj.mclmc.build_kernel()
    step_keys = bj.random.split(key, Tn)
    s, rows, des = st, [], []
    for t in range(Tn):
        s, info = kernel(step_keys[t], s, tgt, imm, L, eps)
        des.append(info.energy_change)
        if (t + 1) % 3 == 0:
            rows.append(s.position)
    torch.cuda.synchronize()
    for a, b in zip(fin, s):
        assert torch.equal(a, b)
    assert torch.equal(hist, torch.stack(rows)) and torch.equal(de, torch.stack(des))
    # two handles of C/2 chains (chain_offset = 0, C/2) give the chains of one handle of C
    halves = []
    for lo in (0, C // 2):
        sub = bj.mcmc.hmc.IntegratorState(*(t[lo:lo + C // 2].clone() for t in st))
        f, _, _ = bj.sample_mclmc_native(key, sub, tgt, L, eps[lo:lo + C // 2].contiguous(), Tn, inverse_mass_matrix=imm,
                                         keep_history=False, chain_offset=lo)
        halves.append(f)
    torch.cuda.synchronize()
    for i in range(4):
        assert torch.equal(torch.cat([halves[0][i], halves[1][i]]), fin[i])


def _bounded():
    return T.UserTarget(2, plugin.read_example("bounded_gaussian"), np.array([5.0], F), name="bounded_gaussian",
                        dense_metric=False, general_integrators=True)


@pytest.mark.parametrize("table, step_size, seeds", [("mclachlan", 100.0, [0]), ("velocity_verlet", 8.0, range(8))])
def test_nan_cases_revert(table, step_size, seeds):
    """test_mclmc_nan_fix_969.py:82-119, one chain per seed: init_key, step_key = split(key(seed))."""
    ks = np.stack([oprng.split(oprng.key(s), 2) for s in seeds])
    init_keys, step_keys = ks[:, 0], ks[:, 1]
    C = len(ks)
    tgt, otgt = _bounded(), otargets.BoundedGaussian(2)
    st = bj.mclmc.init(tf(np.zeros((C, 2))), tgt, tk(init_keys))
    new, info = bj.mclmc.build_kernel(integrator=TABLES[table])(tk(step_keys), st, tgt, 1.0, 1.0, step_size)
    ostate = om.mclmc_init(np.zeros((C, 2), F), otgt, init_keys)
    (oq, ou, ologp, og), oinfo = om.mclmc_kernel(step_keys, ostate, otgt, np.ones(2, F), F(1.0), F(step_size),
                                                 TABLES[table])
    torch.cuda.synchronize()
    assert not npy(info.nonans).any() and not oinfo.nonans.any()
    assert np.all(np.isfinite(npy(new.logdensity))) and np.all(npy(new.position) == 0)
    np.testing.assert_allclose(npy(new.momentum), ou, rtol=0, atol=1e-6)
    assert np.all(npy(info.energy_change) == 0) and np.all(npy(info.kinetic_change) == 0)


def test_unsupported_configurations_are_rejected():
    rs = np.random.default_rng(0)
    key = tk(oprng.key(0))

    def step(tgt, D, imm, C=8):
        st = bj.mclmc.init(tf(rs.standard_normal((C, D))), tgt, key)
        return bj.mclmc.build_kernel()(key, st, tgt, imm, 3.0, 0.5)

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
        with pytest.raises(_lib.BjxError, match="error -2"):
            step(tgt, D, imm)
    eng = bj._engine.get_engine(tf(np.zeros((4, 1))), T.StdNormal(1))
    with pytest.raises(_lib.BjxError, match="error -2: MCLMC needs dim >= 2"):
        eng.mclmc_init(key, tf(np.zeros((4, 1))))


def test_long_run_recovers_gaussian_moments():
    """4096 chains, 600 transitions on a scaled 64-D Gaussian with its own diagonal metric: pooled mean and variance."""
    D, C = 64, 4096
    rs = np.random.default_rng(3)
    s = np.exp(rs.uniform(-1, 1, D))
    tgt = T.DiagGaussian(s)
    key = tk(oprng.key(5))
    st = bj.mclmc.init(tf(rs.standard_normal((C, D))), tgt, key)
    _, hist, de = bj.sample_mclmc_native(key, st, tgt, math.sqrt(D), 0.25 * math.sqrt(D), 600,
                                         inverse_mass_matrix=tf(s * s), thin=10)
    x = npy(hist[20:]).reshape(-1, D) / s
    assert np.all(np.abs(x.mean(0)) < 0.05)
    assert np.all(np.abs(x.var(0) - 1.0) < 0.08)
    assert np.all(np.isfinite(npy(de)))
