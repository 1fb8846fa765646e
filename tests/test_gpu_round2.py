"""GPU parity tests added in round 2 (VERDICT items 2 and 3, ADVICE): the named configurations at their own shapes,
teacher-forced shared adaptation, tie checks for every NUTS chain that disagrees with the oracle, stream and metric-cache
hygiene, and the G = 1 vs G = 2 invariance of the sharded warm-up.  Everything goes through the C ABI (ctypes)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import blackjax_b200 as bj
from blackjax_b200 import _engine, targets as T
from blackjax_b200._lib import check, lib, ptr
from oracle import adaptation as oadapt
from oracle import hmc as ohmc
from oracle import nuts as onuts
from oracle import prng as oprng
from oracle import targets as otargets

pytestmark = pytest.mark.gpu
F = np.float32
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def tk(keys_np):
    return torch.from_numpy(np.ascontiguousarray(keys_np).view(np.int32)).to(DEV).view(torch.uint32)


def tf(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(DEV)


def npy(t):
    return t.detach().cpu().numpy()


def close_elementwise(a, b, rtol, floor):
    """|a - b| <= rtol * max(|b|, floor) for EVERY element: relative to the element itself, with an absolute floor that
    is stated by the caller (the scale below which the quantity is noise for the comparison at hand)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    bound = rtol * np.maximum(np.abs(b), floor)
    bad = np.abs(a - b) > bound
    assert not bad.any(), (f"{bad.sum()} of {bad.size} elements off; worst |a-b|/max(|b|,floor) = "
                           f"{np.max(np.abs(a - b) / np.maximum(np.abs(b), floor)):.3e} (rtol {rtol:.1e}, floor {floor:.1e})")


def max_rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / max(float(np.max(np.abs(b))), 1e-300))


# ---------------------------------------------------------------------------------------------------------
# BASELINE config 2 at its own shape: 1024-D correlated Gaussian, dense mass matrix, 64-chain oracle subset
# ---------------------------------------------------------------------------------------------------------
def test_config2_single_products_within_1e_5():
    """The stated tolerance, on the unit it applies to: ONE float32-accurate product at config 2's matrices (v = M^-1 p,
    g = -P q, p = L^-T z), error / max |y| against float64."""
    C, D = 256, 1024
    cov, prec = otargets.correlated_gaussian(D, seed=0)
    tgt = T.DenseGaussian(prec)
    eng = _engine.Engine(DEV, C, D, tgt)
    eng.set_metric(tf(cov))
    rs = np.random.default_rng(8)
    p = rs.standard_normal((C, D)).astype(F)
    q = (0.1 * rs.standard_normal((C, D))).astype(F)
    v = npy(eng.velocity(tf(p)))
    _, g = eng.init_state(tf(q))
    e_v = max_rel(v, p.astype(np.float64) @ cov.astype(np.float64))
    e_g = max_rel(npy(g), -(q.astype(np.float64) @ prec.astype(np.float64)))
    keys = oprng.split(oprng.key(2), C)
    mom = npy(eng.sample_momentum(tk(keys)))
    e_m = max_rel(mom, ohmc.Metric(cov).sample_momentum(keys, D))
    print(f"single products at config 2: velocity {e_v:.2e} gradient {e_g:.2e} momentum {e_m:.2e}")
    assert e_v < 1e-5 and e_g < 1e-5 and e_m < 1e-5
    eng.close()


@pytest.mark.parametrize("L, tol_q, tol_p, tol_energy", [(1, 3e-5, 1e-5, 1e-5), (5, 4e-5, 4e-5, 1e-5), (50, 3e-3, 1e-4, 1e-5)])
def test_config2_dense_1024_transition_vs_oracle(L, tol_q, tol_p, tol_energy):
    """Full HMC transition at config 2's matrices (Sigma = Q diag(logspace(-1,1)) Q^T, kappa = 100, M^-1 = Sigma, eps = 0.5)
    against the float32 oracle from the same (state, key), error / max |reference|.
    The stated tolerance of the path is 1e-5 per float32 product (test_config2_single_products_within_1e_5).  Whatever
    error the tensor core's float32 accumulation over 3K/16 = 192 steps leaves acts like a small change of M^-1 and P,
    i.e. of the oscillation frequencies.  Energies, momenta and the accept decision are insensitive to it; the POSITION of
    the stiffest modes at eps = 0.5 (phase advance per step close to the stability limit) accumulates it as a phase shift
    that grows with L (two exact float32 implementations would already differ by ~1e-4 after 50 steps).  At L = 1 the
    momentum draw, the first half kick's gradient and M^-1 p are three products whose errors add."""
    C, D = 64, 1024
    cov, prec = otargets.correlated_gaussian(D, seed=0)
    tgt, otgt = T.DenseGaussian(prec), otargets.DenseGaussian(prec)
    rs = np.random.default_rng(4)
    q = (0.1 * rs.standard_normal((C, D))).astype(F)
    keys = oprng.split(oprng.key(23), C)
    onew, oinfo = ohmc.hmc_kernel(keys, ohmc.init(q, otgt), otgt, F(0.5), ohmc.Metric(cov), L)
    new, info = bj.hmc.build_kernel(full_info=True)(tk(keys), bj.hmc.init(tf(q), tgt), tgt, 0.5, tf(cov), L)
    torch.cuda.synchronize()
    e_mom = max_rel(npy(info.momentum), oinfo.momentum)
    e_q = max_rel(npy(info.proposal.position), oinfo.proposal[0])
    e_p = max_rel(npy(info.proposal.momentum), oinfo.proposal[1])
    e_en = float(np.max(np.abs(npy(info.energy) - oinfo.energy)) / (np.max(np.abs(oinfo.energy)) + D))
    print(f"config-2 shape, L={L}: momentum {e_mom:.2e}  proposal q {e_q:.2e} p {e_p:.2e}  energy {e_en:.2e}")
    assert e_mom < 1e-5
    assert e_q < tol_q and e_p < tol_p
    assert e_en < tol_energy
    u = oprng.uniform(oprng.split(keys, 2)[:, 1])
    acc = npy(info.is_accepted)
    # a differing accept decision must sit on a tie: |u - p_accept| below the acceptance-rate error the energy error allows
    tie = np.abs(u - oinfo.acceptance_rate) < 5 * tol_energy * (np.max(np.abs(oinfo.energy)) + D)   # d p_accept <= d energy
    assert ((acc == oinfo.is_accepted) | tie).all()


# ---------------------------------------------------------------------------------------------------------
# BASELINE config 4's adaptation path: D = 512 shared warm-up, teacher-forced per step against oracle/adaptation.py
# ---------------------------------------------------------------------------------------------------------
def test_config4_shared_adaptation_teacher_forced_d512():
    """Every warm-up step, the device update (bjx_adapt_shared_update: block statistics -> merge -> dual averaging ->
    window bookkeeping) and the oracle (staged_adaptation.py:153-171,233-297 restated) are fed the SAME positions and
    acceptance rates; step size after every step, inverse mass matrix at the window end and the final step size must
    agree to 1e-5 relative (elementwise; the inverse mass matrix has no small elements: floor = its smallest entry)."""
    D, C, T_ = 512, 8192, 150          # two statistic blocks; schedule: 75 fast, one 25-step slow window, 50 fast
    scale = np.logspace(-1, 1, D)
    tgt = T.DiagGaussian(scale)
    rs = np.random.default_rng(12)
    q = rs.standard_normal((C, D)).astype(F)
    state = bj.nuts.init(tf(q), tgt)
    eng = _engine.get_engine(state.position, tgt, max_tree_depth=6)
    kernel = bj.nuts.build_kernel(max_tree_depth=6)
    L_ = lib()
    st = torch.empty(L_.bjx_adapt_shared_state_floats(C, D, 1), device=DEV)
    eps_c = torch.empty(C, device=DEV)
    imm = torch.empty(D, device=DEV)
    hist = torch.empty(T_, device=DEV)
    check(L_.bjx_adapt_shared_init(eng.h, ptr(st), 1.0, ptr(eps_c), ptr(imm)), eng.h)
    eng._imm, eng._imm_key = imm, (imm.data_ptr(), tuple(imm.shape), imm._version, str(imm.device))
    oda, owf, oimm = oadapt.da_init(1.0), oadapt.welford_init(D), np.ones(D, F)
    step_keys = bj.random.split(bj.random.key(3, DEV), T_)
    schedule = oadapt.build_schedule(T_)
    assert any(w for _, w in schedule)
    for t, (stage, wend) in enumerate(schedule):
        state, info = kernel(step_keys[t], state, tgt, eps_c, imm, 6)
        check(L_.bjx_adapt_shared_update(eng.h, None, 1, ptr(st), ptr(state.position), ptr(info.acceptance_rate),
                                         int(stage), int(wend), 0.8, ptr(eps_c), ptr(imm), ptr(hist)), eng.h)
        x, a = npy(state.position), npy(info.acceptance_rate)
        if stage == 1:
            mean_b = np.mean(x, axis=0, dtype=F)
            cb = (x - mean_b).astype(F)
            owf = oadapt.cgl_merge(owf, oadapt.Welford(mean_b, np.sum(cb * cb, axis=0, dtype=F), C))
        oda = oadapt.da_update(oda, np.mean(a, dtype=F), 0.8)
        oeps = np.exp(oda.log_step_size).astype(F)
        if wend:
            oimm = oadapt.welford_final(owf)
            owf = oadapt.welford_init(D)
            oda = oadapt.da_init(oadapt.da_final(oda))
            oeps = np.exp(oda.log_step_size).astype(F)
            close_elementwise(npy(imm), oimm, rtol=1e-5, floor=float(oimm.min()))
        dev_eps = npy(eps_c)
        assert (dev_eps == dev_eps[0]).all()                       # one step size for all chains
        close_elementwise(dev_eps[:1], [oeps], rtol=1e-5, floor=1e-30)
    close_elementwise(npy(hist)[-1:], [oeps], rtol=1e-5, floor=1e-30)
    fin = torch.empty(1, device=DEV)
    check(L_.bjx_adapt_shared_final(eng.h, ptr(st), ptr(fin)), eng.h)
    close_elementwise(npy(fin), [oadapt.da_final(oda)], rtol=1e-5, floor=1e-30)
    # the adapted metric tracks the target's variances (25 pooled draws x 8192 chains)
    np.testing.assert_allclose(npy(imm), scale ** 2, rtol=0.25)


def test_packaged_shared_warmup_equals_the_teacher_forced_loop_and_old_python_path():
    """window_adaptation(shared=True).run is exactly the loop above (same bits), and the device-side merge / dual
    averaging agrees with the host-side float32 restatement it replaced to 1e-5 on a free run of 60 steps."""
    D, C, T_ = 64, 4096 + 1024, 60     # a full and a partial statistic block
    scale = np.logspace(-0.5, 0.5, D)
    tgt = T.DiagGaussian(scale)
    q = np.random.default_rng(5).standard_normal((C, D)).astype(F)
    warm = bj.window_adaptation(bj.hmc, tgt, shared=True, num_integration_steps=8)
    (st, params), hist = warm.run(bj.random.key(9, DEV), tf(q), T_)
    (st2, params2), hist2 = warm.run(bj.random.key(9, DEV), tf(q), T_)
    assert torch.equal(st.position, st2.position) and params["step_size"] == params2["step_size"]
    assert torch.equal(params["inverse_mass_matrix"], params2["inverse_mass_matrix"])
    okern = lambda k, s, t, e, m, **kw: ohmc.hmc_kernel(k, s, t, e, m, 8)
    ost, oeps, oimm, ohist = oadapt.window_adaptation_run(okern, otargets.DiagGaussian(scale), oprng.key(9), q, T_, shared=True)
    np.testing.assert_allclose(np.asarray(hist)[:15], ohist[:15], rtol=2e-4)   # free-running: accept flips on ties later on
    assert abs(params["step_size"] / float(oeps) - 1) < 0.05


# ---------------------------------------------------------------------------------------------------------
# NUTS: every chain that disagrees with the oracle sits on a float tie
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind, D, C, depth, eps", [("funnel", 128, 1024, 10, 0.1), ("diag", 64, 512, 8, 0.3),
                                                    ("std", 100, 512, 6, 0.4)])
def test_nuts_disagreements_sit_on_ties(kind, D, C, depth, eps):
    rs = np.random.default_rng(41)
    if kind == "funnel":
        tgt, otgt = T.Funnel(D), otargets.Funnel(D)
        q = (0.1 * rs.standard_normal((C, D))).astype(F)
    elif kind == "diag":
        s = np.exp(rs.uniform(-1, 1, D))
        tgt, otgt = T.DiagGaussian(s), otargets.DiagGaussian(s)
        q = (rs.standard_normal((C, D)) * s).astype(F)
    else:
        tgt, otgt = T.StdNormal(D), otargets.StdNormal(D)
        q = rs.standard_normal((C, D)).astype(F)
    imm = np.ones(D, F)
    keys = oprng.split(oprng.key(77), C)
    margins = np.full(C, np.inf)
    onew, oinfo = onuts.nuts_kernel(keys, ohmc.init(q, otgt), otgt, F(eps), imm, depth, margins=margins)
    new, info = bj.nuts.build_kernel(max_tree_depth=depth)(tk(keys), bj.nuts.init(tf(q), tgt), tgt, eps, tf(imm), depth)
    torch.cuda.synchronize()
    same = ((npy(info.num_integration_steps) == oinfo.num_integration_steps)
            & (npy(info.num_trajectory_expansions) == oinfo.num_trajectory_expansions)
            & (npy(info.is_turning) == oinfo.is_turning) & (npy(info.is_divergent) == oinfo.is_divergent)
            & np.all(np.isclose(npy(new.position), onew.position, rtol=1e-4, atol=1e-5), axis=1))
    print(f"{kind} D={D}: {same.mean():.4f} of chains identical; margins of the others: {np.sort(margins[~same])[:6]}; "
          f"max tree {oinfo.num_integration_steps.max()}")
    assert same.mean() >= 0.97
    # One transition integrates up to 2^depth leapfrogs from an identical start; device and oracle differ by float32
    # rounding (<= 1e-6 relative per leapfrog, growing along the trajectory), so a chain can only take another branch if
    # one of the oracle's decisions on its path was closer to its boundary than that accumulated difference: 1e-5
    # relative per the stated tolerance, times the trajectory length headroom below.
    assert (margins[~same] < 1e-5 * 64).all(), np.sort(margins[~same])[-3:]
    # and the converse sanity check: chains far from every boundary agree
    assert same[margins > 1e-2].all()


def test_nuts_runs_without_host_round_trips_and_reports_depth_on_request():
    C, D = 4096, 32
    tgt = T.Funnel(D)
    st = bj.nuts.init(0.1 * torch.randn(C, D, device=DEV), tgt)
    kern = bj.nuts.build_kernel()
    keys = bj.random.split(bj.random.key(2, DEV), 3)
    for k in keys:
        st, info = kern(k, st, tgt, 0.2, torch.ones(D, device=DEV), 10)
    eng = _engine.get_engine(st.position, tgt)
    launches, depth = eng.nuts_last_stats()
    assert launches == 1 + (10 - 4)                            # fused doublings 0-3, then one launch per further doubling
    assert depth == int(info.num_trajectory_expansions.max())


# ---------------------------------------------------------------------------------------------------------
# ADVICE: PRNG calls on side streams; metric cache keyed on content version
# ---------------------------------------------------------------------------------------------------------
def test_prng_and_warmup_inside_a_side_stream():
    s = torch.cuda.Stream(device=DEV)
    tgt = T.DiagGaussian(np.logspace(-0.3, 0.3, 16))
    q = torch.randn(512, 16, device=DEV)
    ref_keys = bj.random.split(bj.random.key(4, DEV), 40)
    warm = bj.window_adaptation(bj.hmc, tgt, num_integration_steps=5)
    (ref_state, ref_params), _ = warm.run(bj.random.key(4, DEV), q, 40)
    alg = bj.dhmc(tgt, 0.3, torch.ones(16, device=DEV))
    ref_d = alg.init(q, bj.random.key(8, DEV))
    for k in ref_keys[:5]:
        ref_d, _ = alg.step(k, ref_d)
    torch.cuda.synchronize()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        # a long kernel first, so that work issued on the legacy default stream would overtake this stream
        junk = torch.randn(4096, 4096, device=DEV) @ torch.randn(4096, 4096, device=DEV)
        keys = bj.random.split(bj.random.key(4, DEV), 40)
        (state, params), _ = warm.run(bj.random.key(4, DEV), q, 40)
        d = alg.init(q, bj.random.key(8, DEV))
        for k in keys[:5]:
            d, _ = alg.step(k, d)
    s.synchronize()
    assert torch.equal(keys, ref_keys)
    assert torch.equal(state.position, ref_state.position)
    assert torch.equal(params["step_size"], ref_params["step_size"])
    assert torch.equal(d.position, ref_d.position)
    del junk


@pytest.mark.parametrize("D, dense", [(16, False), (256, True)])
def test_inplace_metric_update_is_picked_up(D, dense):
    C = 64
    rs = np.random.default_rng(2)
    if dense:
        A = rs.standard_normal((D, D))
        imm_a = (A @ A.T / D + np.eye(D)).astype(F)
        imm_b = (2.5 * imm_a).astype(F)
    else:
        imm_a, imm_b = np.exp(rs.uniform(-1, 1, D)).astype(F), np.exp(rs.uniform(-1, 1, D)).astype(F)
    tgt = T.DiagGaussian(np.ones(D, F))
    q = tf(rs.standard_normal((C, D)))
    key = bj.random.key(1, DEV)
    kern = bj.hmc.build_kernel(full_info=True)
    imm = tf(imm_a)
    _, info_a = kern(key, bj.hmc.init(q, tgt), tgt, 0.1, imm, 3)
    imm.copy_(tf(imm_b))                                        # same tensor, new contents
    _, info_b = kern(key, bj.hmc.init(q, tgt), tgt, 0.1, imm, 3)
    _, info_ref = kern(key, bj.hmc.init(q, tgt), tgt, 0.1, tf(imm_b), 3)
    assert not torch.equal(info_a.momentum, info_b.momentum)
    assert torch.equal(info_b.momentum, info_ref.momentum)      # mass_matrix_sqrt / operand planes were re-derived
    assert torch.equal(info_b.proposal.position, info_ref.proposal.position)


# ---------------------------------------------------------------------------------------------------------
# the sharded warm-up does not depend on the GPU count (needs two GPUs: `gpurun --gpus 2`)
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs (gpurun --gpus 2)")
def test_shared_warmup_bit_identical_on_one_and_two_gpus(tmp_path):
    worker = os.path.join(ROOT, "tests", "helpers", "shared_warmup_worker.py")
    one, two = str(tmp_path / "g1.npz"), str(tmp_path / "g2.npz")
    env = dict(os.environ, PYTHONPATH=ROOT)
    subprocess.run([sys.executable, worker, one, "16384"], check=True, env=env, timeout=600)
    subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
                    "127.0.0.1", "--master-port", "29517", worker, two, "8192"], check=True, env=env, timeout=600)
    a, b = np.load(one), np.load(two)
    assert a["n_ranks"] == 1 and b["n_ranks"] == 2
    for k in ("eps_history", "imm", "step_size", "position", "logdensity"):
        assert np.array_equal(a[k], b[k]), k


# ---------------------------------------------------------------------------------------------------------
# config 5: the fast sigmoid / softplus (ex2.approx, rcp, lg2.approx) against float64
# ---------------------------------------------------------------------------------------------------------
def test_hier_logit_fast_math_error_bounds():
    """value_and_grad of the hierarchical logistic regression with one exponential, one reciprocal and one logarithm per
    observation (bjx_big.cu) against a float64 evaluation of the same formulas: per-group gradient entries (sums of 8
    sigmoids) within 4e-6 absolute, log-density within 1e-6 of the sum of its term magnitudes, including saturated
    observations (|eta| up to ~40)."""
    D, C = 2052, 12
    G = D - 4
    x, bits = T.HierLogit.synthetic_data(G, seed=3)
    tgt = T.HierLogit(x, bits)
    rs = np.random.default_rng(0)
    q = np.zeros((C, D), F)
    q[:, 0], q[:, 1], q[:, 2], q[:, 3] = 0.5, np.log(0.7), 1.0, -0.5
    q[:, 4:] = (0.5 + 0.7 * rs.standard_normal((C, G))).astype(F)
    q[C // 2:, 4:] *= 25.0                       # saturated logits in half of the chains
    eng = _engine.Engine(DEV, C, D, tgt)
    logp, g = eng.init_state(tf(q))
    q64 = q.astype(np.float64)
    xs = np.asarray(x, np.float64)
    y = ((np.asarray(bits, np.uint8)[:, None] >> np.arange(8, dtype=np.uint8)) & 1).astype(np.float64)
    mu, lt, b0, b1, alpha = q64[:, 0], q64[:, 1], q64[:, 2], q64[:, 3], q64[:, 4:]
    eta = alpha[:, :, None] + b0[:, None, None] * xs[None, :, :, 0] + b1[:, None, None] * xs[None, :, :, 1]
    sig = 1.0 / (1.0 + np.exp(-eta))
    softplus = np.maximum(eta, 0.0) + np.log1p(np.exp(-np.abs(eta)))
    e2 = np.exp(-2.0 * lt)
    d = alpha - mu[:, None]
    ll = np.sum(y * eta - softplus, axis=(1, 2))
    ref_logp = -0.005 * mu ** 2 - 0.5 * lt ** 2 - 0.08 * (b0 ** 2 + b1 ** 2) + (-0.5 * e2 * np.sum(d * d, 1) - G * lt) + ll
    ref_ga = -d * e2[:, None] + np.sum(y - sig, axis=2)
    terms = np.sum(np.abs(y * eta) + softplus, axis=(1, 2)) + 0.5 * e2 * np.sum(d * d, 1)
    assert np.max(np.abs(npy(logp) - ref_logp) / terms) < 1e-6
    ga = npy(g)[:, 4:]
    # the prior part -d e2 is exact float32 arithmetic (relative 1e-6 of its size); the likelihood part is 8 fast sigmoids
    assert np.max(np.abs(ga - ref_ga) / (1.0 + np.abs(d * e2[:, None]))) < 4e-6
    gb = npy(g)[:, 2]
    ref_gb = -0.16 * b0 + np.sum((y - sig) * xs[None, :, :, 0], axis=(1, 2))
    assert np.max(np.abs(gb - ref_gb)) / np.sum(np.abs(xs[:, :, 0])) < 1e-6
    eng.close()


# ---------------------------------------------------------------------------------------------------------
# SURVEY 8f item 4: ChEES-HMC warm-up (blackjax/adaptation/chees_adaptation.py), device update vs oracle/chees.py
# ---------------------------------------------------------------------------------------------------------
def test_chees_update_teacher_forced_vs_oracle():
    """Every warm-up step the device update (bjx_chees_update) and the oracle's chees_update are fed the SAME transition
    (initial positions, proposals, acceptance probabilities, divergence flags): step size, trajectory length and the next
    step count must agree (1e-5 relative; the step count exactly unless jitter*T/eps sits within 1e-5 of an integer)."""
    from oracle import chees as ochees
    D, C, T_ = 24, 4096 + 512, 60
    scale = np.logspace(-0.5, 1.0, D)
    tgt = T.DiagGaussian(scale)
    q = (np.random.default_rng(2).standard_normal((C, D)) * scale).astype(F)
    kernel = bj.hmc.build_kernel(full_info=True)
    state = bj.hmc.init(tf(q), tgt)
    eng = _engine.get_engine(state.position, tgt)
    L_ = lib()
    max_bits = 11
    st = torch.empty(L_.bjx_chees_state_floats(C, D, 1), device=DEV)
    eps_c = torch.empty(C, device=DEV)
    steps_c = torch.empty(C, dtype=torch.int32, device=DEV)
    check(L_.bjx_chees_init(eng.h, ptr(st), 0.05, max_bits, 1.0, ptr(eps_c), ptr(steps_c)), eng.h)
    imm = torch.ones(D, device=DEV)
    os_ = ochees.chees_init(0.05)
    keys = bj.random.split(bj.random.key(5, DEV), T_)
    for t in range(T_):
        L_dev = int(steps_c[0])
        L_or = ochees.integration_steps(os_.random_generator_arg, F(os_.trajectory_length / os_.step_size), 1.0, max_bits)
        x = float(ochees.jitter(os_.random_generator_arg, 1.0, max_bits)) * float(os_.trajectory_length / os_.step_size)
        assert L_dev == L_or or abs(x - round(x)) < 1e-4 * max(x, 1.0), (t, L_dev, L_or, x)
        assert bool((steps_c == L_dev).all()) and bool((eps_c == eps_c[0]).all())
        init_q = state.position
        state, info = kernel(keys[t], state, tgt, eps_c, imm, steps_c)
        div = info.is_divergent.to(torch.uint8)
        check(L_.bjx_chees_update(eng.h, None, 1, ptr(st), ptr(init_q), ptr(info.proposal.position), ptr(info.proposal.momentum),
                                  ptr(info.acceptance_rate), ptr(div), 0.1, 0.9, 0.999, 0.651, 0.5, 1000, ptr(eps_c),
                                  ptr(steps_c), None), eng.h)
        os_ = ochees.chees_update(os_, npy(info.proposal.position), npy(info.proposal.momentum), npy(init_q),
                                  npy(info.acceptance_rate), npy(info.is_divergent), lr=0.1, max_bits=max_bits)
        hdr = npy(st[:16])
        close_elementwise(hdr[[0, 2]], [os_.step_size, os_.trajectory_length], rtol=1e-5, floor=1e-30)
        close_elementwise(hdr[[1, 3]], [os_.log_step_size_ma, os_.log_trajectory_length_ma], rtol=2e-5, floor=1e-2)
        # teacher forcing: continue from the oracle's state bits so that rounding differences cannot accumulate
        st[0], st[1], st[2], st[3] = float(os_.step_size), float(os_.log_step_size_ma), float(os_.trajectory_length), float(os_.log_trajectory_length_ma)
        st[4], st[5], st[7] = float(os_.da.log_step_size), float(os_.da.log_step_size_avg), float(os_.da.avg_error)
        st[10], st[11] = float(os_.optim.mu), float(os_.optim.nu)
    assert float(os_.trajectory_length) > 3 * float(os_.step_size)     # the criterion did lengthen the trajectories


def test_chees_adaptation_reference_test_problem():
    """tests/adaptation/test_adaptation.py:77-140 of the reference: 2-D normal with std (1, 10), step size 0.1,
    adam(learning_rate=0.5, b1=0, b2=0.95), target acceptance 0.75; after the warm-up, dynamic HMC with the adapted
    parameters must show a harmonic-mean acceptance near the target and recover the target's scales.  More chains than
    the reference's 16 (the statistics are pooled over chains; 16 chains make the comparison with the oracle's free run
    noisy), same schedule."""
    from blackjax_b200.adaptation.chees_adaptation import adam
    from oracle import chees as ochees
    C, burn = 512, 400
    std = np.array([1.0, 10.0])
    tgt, otgt = T.DiagGaussian(std), otargets.DiagGaussian(std)
    q = np.random.default_rng(1).standard_normal((C, 2)).astype(F)
    warm = bj.chees_adaptation(tgt, num_chains=C, target_acceptance_rate=0.75)
    (last, params), hist = warm.run(bj.random.key(346, DEV), tf(q), step_size=0.1, optim=adam(0.5, b1=0.0, b2=0.95), num_steps=burn)
    ost, oeps, onlf, os_ = ochees.chees_run(otgt, oprng.key(346), q, 0.1, lr=0.5, b1=0.0, b2=0.95, num_steps=burn,
                                            target_acceptance_rate=0.75)
    print(f"ChEES: device eps {params['step_size']:.4f} L {params['integration_steps_params'][0]:.2f}; "
          f"oracle eps {float(oeps):.4f} L {float(onlf):.2f}")
    assert abs(params["step_size"] / float(oeps) - 1) < 0.15
    assert abs(params["integration_steps_params"][0] / float(onlf) - 1) < 0.3
    alg = bj.dhmc(tgt, **params)
    state = last
    keys = bj.random.split(bj.random.key(9, DEV), 200)
    inv_acc, draws = [], []
    for k in keys:
        state, info = alg.step(k, state)
        inv_acc.append((1.0 / info.acceptance_rate).mean())
        draws.append(state.position)
    hm = float((1.0 / torch.stack(inv_acc)).mean())
    assert abs(hm - 0.75) < 0.1, hm
    x = torch.stack(draws[50:]).reshape(-1, 2)
    np.testing.assert_allclose(npy(x.std(0)), std, rtol=0.15)


@pytest.mark.parametrize("C,D,T_,depth,thin,metric", [(2048, 32, 6, 8, 1, "diag"), (301, 256, 5, 6, 2, "diag"),
                                                       (512, 16, 4, 7, 1, "dense"), (1000, 128, 3, 5, 1, "diag")])
def test_native_nuts_sampler_equals_stepwise_calls(C, D, T_, depth, thin, metric):
    """bjx_nuts_sample (run_inference_algorithm for NUTS without a Python loop) gives the draws of T calls of nuts.step,
    bit for bit -- with T >= 4 through the decoupled-chains kernel (k_nuts_chains: every warp takes whole chains through
    all transitions), below that through the step-synchronous loop."""
    tgt = T.Funnel(D)
    g = torch.Generator(device=DEV).manual_seed(C)
    q = 0.1 * torch.randn(C, D, device=DEV, generator=g)
    if metric == "dense":
        a = torch.randn(D, D, device=DEV, generator=g) * 0.2
        imm = a @ a.T + torch.eye(D, device=DEV)
    else:
        imm = torch.exp(0.3 * torch.randn(D, device=DEV, generator=g))
    st0 = bj.nuts.init(q, tgt)
    key = bj.random.key(12, DEV)
    fin, hist, acc, n_int = bj.sample_nuts_native(key, st0, tgt, 0.2, imm, T_, max_num_doublings=depth, thin=thin)
    alg = bj.nuts(tgt, 0.2, imm, max_num_doublings=depth)
    st = alg.init(q)
    keys = bj.random.split(key, T_)
    for t in range(T_):
        st, info = alg.step(keys[t], st)
        if (t + 1) % thin == 0:
            assert torch.equal(hist[(t + 1) // thin - 1], st.position)
        assert torch.equal(n_int[t], info.num_integration_steps) and torch.equal(acc[t], info.acceptance_rate)
    assert hist.shape[0] == T_ // thin
    assert torch.equal(fin.position, st.position) and torch.equal(fin.logdensity, st.logdensity)
    assert torch.equal(fin.logdensity_grad, st.logdensity_grad)


def test_dense_shared_window_adaptation_d256_recovers_covariance():
    """welford_dense recipe, chain-pooled, at dim > 128 (mass_matrix.py:411-442, metric_buffers.py:396-420): HMC on the
    tensor-core dense path, the D x D co-moment block from bjx_pooled_stats_dense against float64 numpy, and the adapted
    dense inverse mass matrix against the target covariance."""
    D, C, T_ = 256, 4096, 150
    rs = np.random.default_rng(3)
    A = rs.standard_normal((D, D)) / np.sqrt(D)
    cov = A @ A.T + 0.5 * np.eye(D)
    tgt = T.DenseGaussian(np.linalg.inv(cov))
    q = rs.standard_normal((C, D)).astype(F)
    warm = bj.window_adaptation(bj.hmc, tgt, is_mass_matrix_diagonal=False, shared=True, num_integration_steps=12)
    (st, params), hist = warm.run(bj.random.key(6, DEV), tf(q), T_)
    imm = npy(params["inverse_mass_matrix"])
    assert imm.shape == (D, D)
    err = np.abs(imm - cov).max() / np.abs(cov).max()
    print(f"dense shared adaptation D=256: max |imm - cov| / max|cov| = {err:.3f}, step size {params['step_size']:.3f}")
    assert err < 0.12                               # 25 pooled draws x 4096 chains
    eng = _engine.get_engine(st.position, tgt)
    out = torch.empty(2 + D + D * D, device=DEV)
    acc = torch.rand(C, device=DEV)
    check(lib().bjx_pooled_stats_dense(eng.h, ptr(st.position), ptr(acc), ptr(out)), eng.h)
    x = npy(st.position).astype(np.float64)
    o = npy(out)
    ref = (x - x.mean(0)).T @ (x - x.mean(0))
    assert np.max(np.abs(o[2:2 + D] - x.mean(0))) < 1e-5 * np.abs(x).max()
    assert np.max(np.abs(o[2 + D:].reshape(D, D) - ref)) < 1e-4 * np.abs(ref).max()


def test_dense_shared_window_adaptation_with_nuts_beyond_128_dims():
    """The welford_dense recipe with NUTS at dim > 128 (every warm-up transition runs on the tensor-core dense path):
    the adapted dense inverse mass matrix approaches the target covariance and the step size is sane."""
    rs = np.random.default_rng(12)
    D, C, T_ = 160, 2048, 150
    a = rs.standard_normal((D, D)) / np.sqrt(D)
    cov = (a @ a.T + 0.3 * np.eye(D))
    prec = np.linalg.inv(cov)
    tgt = T.DenseGaussian((0.5 * (prec + prec.T)).astype(F))
    q = rs.standard_normal((C, D)).astype(F)
    warm = bj.window_adaptation(bj.nuts, tgt, is_mass_matrix_diagonal=False, shared=True, max_num_doublings=5)
    (st, params), hist = warm.run(bj.random.key(3, DEV), tf(q), T_)
    imm = npy(params["inverse_mass_matrix"])
    err = np.abs(imm - cov).max() / np.abs(cov).max()
    print(f"dense shared NUTS adaptation D={D}: max |imm - cov| / max|cov| = {err:.3f}, step size {params['step_size']:.3f}")
    assert imm.shape == (D, D) and np.isfinite(imm).all()
    assert err < 0.2 and 0.05 < params["step_size"] < 2.0


# ---------------------------------------------------------------------------------------------------------
# SURVEY 8f item 4: the low-rank metric (blackjax/mcmc/metrics.py:349-467) in the warp kernels
# ---------------------------------------------------------------------------------------------------------
def _low_rank_problem(D, k, seed):
    rs = np.random.default_rng(seed)
    U, _ = np.linalg.qr(rs.standard_normal((D, k)))
    sigma = np.exp(rs.uniform(-0.7, 0.7, D)).astype(F)
    lam = np.exp(rs.uniform(-1.5, 1.5, k)).astype(F)
    return sigma, U.astype(F), lam


@pytest.mark.parametrize("kind, D, k, C, L", [("diag", 64, 3, 48, 7), ("funnel", 128, 8, 40, 6), ("diag", 256, 16, 33, 5),
                                              ("diag", 512, 5, 24, 4)])
def test_low_rank_metric_hmc_matches_oracle(kind, D, k, C, L):
    from blackjax_b200.mcmc.metrics import gaussian_euclidean_low_rank
    sigma, U, lam = _low_rank_problem(D, k, 7)
    rs = np.random.default_rng(8)
    if kind == "funnel":
        tgt, otgt = T.Funnel(D), otargets.Funnel(D)
        q = (0.2 * rs.standard_normal((C, D))).astype(F)
    else:
        s = np.exp(rs.uniform(-0.5, 0.5, D))
        tgt, otgt = T.DiagGaussian(s), otargets.DiagGaussian(s)
        q = (rs.standard_normal((C, D)) * s).astype(F)
    metric = gaussian_euclidean_low_rank(tf(sigma), tf(U), tf(lam))
    ometric = ohmc.LowRankMetric(sigma, U, lam)
    keys = oprng.split(oprng.key(31), C)
    onew, oinfo = ohmc.hmc_kernel(keys, ohmc.init(q, otgt), otgt, F(0.05), ometric, L)
    new, info = bj.hmc.build_kernel(full_info=True)(tk(keys), bj.hmc.init(tf(q), tgt), tgt, 0.05, metric, L)
    torch.cuda.synchronize()
    from test_gpu_parity import close
    close(npy(info.momentum), oinfo.momentum, rtol=1e-5)
    close(npy(info.proposal.position), oinfo.proposal[0], rtol=2e-5)
    close(npy(info.proposal.momentum), oinfo.proposal[1], rtol=2e-5)
    close(npy(info.energy), oinfo.energy, rtol=1e-5, scale=np.max(np.abs(oinfo.energy)) + D)
    u = oprng.uniform(oprng.split(keys, 2)[:, 1])
    assert ((npy(info.is_accepted) == oinfo.is_accepted) | (np.abs(u - oinfo.acceptance_rate) < 1e-4)).all()
    # the momentum draw has covariance M = (M^-1)^-1
    if D == 64:
        eng = _engine.get_engine(new.position, tgt)
        big = _engine.Engine(DEV, 20000, D, tgt)
        big.ensure_metric(metric)
        p = npy(big.sample_momentum(bj.random.split(bj.random.key(4, DEV), 20000)))
        Minv = np.diag(sigma) @ (np.eye(D) + U @ np.diag(lam - 1) @ U.T) @ np.diag(sigma)
        M = np.linalg.inv(Minv.astype(np.float64))
        assert np.abs(np.cov(p.T) - M).max() < 0.08 * np.abs(M).max()
        big.close()


def test_low_rank_metric_nuts_matches_oracle():
    from blackjax_b200.mcmc.metrics import gaussian_euclidean_low_rank
    D, k, C = 96, 4, 256
    sigma, U, lam = _low_rank_problem(D, k, 9)
    s = np.exp(np.random.default_rng(1).uniform(-0.5, 0.5, D))
    tgt, otgt = T.DiagGaussian(s), otargets.DiagGaussian(s)
    q = (np.random.default_rng(2).standard_normal((C, D)) * s).astype(F)
    keys = oprng.split(oprng.key(13), C)
    margins = np.full(C, np.inf)
    onew, oinfo = onuts.nuts_kernel(keys, ohmc.init(q, otgt), otgt, F(0.2), ohmc.LowRankMetric(sigma, U, lam), 7, margins=margins)
    metric = gaussian_euclidean_low_rank(tf(sigma), tf(U), tf(lam))
    new, info = bj.nuts.build_kernel(max_tree_depth=7)(tk(keys), bj.nuts.init(tf(q), tgt), tgt, 0.2, metric, 7)
    torch.cuda.synchronize()
    same = ((npy(info.num_integration_steps) == oinfo.num_integration_steps) & (npy(info.is_turning) == oinfo.is_turning)
            & np.all(np.isclose(npy(new.position), onew.position, rtol=1e-4, atol=1e-5), axis=1))
    print(f"low-rank NUTS: {same.mean():.4f} identical; margins of the others {np.sort(margins[~same])[:5]}")
    assert same.mean() >= 0.97
    assert (margins[~same] < 1e-5 * 64).all()
    assert oinfo.num_integration_steps.max() >= 15


@pytest.mark.parametrize("metric,target,D,C,depth,eps", [("dense", "diag", 256, 96, 5, 0.35), ("dense", "dense", 256, 64, 5, 0.3),
                                                          ("diag", "dense", 192, 64, 4, 0.3), ("dense", "dense", 512, 32, 6, 0.25)])
def test_dense_path_nuts_matches_oracle(metric, target, D, C, depth, eps):
    """NUTS beyond 128 dims with a dense metric and / or a dense Gaussian target (lock-step leaves on the tensor-core
    products, bjx_dense_nuts.cuh) against the oracle: tree sizes, depths, flags and positions agree except for chains one
    of whose decisions sat on a float tie (the products are good to ~2e-6, so the tie window is wider than for the warp
    kernels' bit-faithful arithmetic)."""
    rs = np.random.default_rng(D + C)
    a = rs.standard_normal((D, D)) / np.sqrt(D)
    cov = (a @ a.T + 0.5 * np.eye(D)).astype(np.float64)
    if target == "dense":
        prec = np.linalg.inv(cov)
        prec = (0.5 * (prec + prec.T)).astype(F)
        tgt, otgt = T.DenseGaussian(prec), otargets.DenseGaussian(prec)
        q = (rs.standard_normal((C, D)) @ np.linalg.cholesky(cov).T).astype(F)
    else:
        s = np.exp(rs.uniform(-0.5, 0.5, D))
        tgt, otgt = T.DiagGaussian(s), otargets.DiagGaussian(s)
        q = (rs.standard_normal((C, D)) * s).astype(F)
    if metric == "dense":
        b = rs.standard_normal((D, D)) / np.sqrt(D)
        imm = (0.3 * (b @ b.T) + np.eye(D)).astype(F)
        imm = (0.5 * (imm + imm.T)).astype(F)
    else:
        imm = np.exp(rs.uniform(-0.3, 0.3, D)).astype(F)
    keys = oprng.split(oprng.key(5), C)
    margins = np.full(C, np.inf)
    # one step size per chain, from tiny (the tree runs to max depth) to unstable (early U-turns inside sub-trees,
    # divergences for the chains started far out in the tail)
    eps_c = (eps * np.logspace(-1.3, 0.9, C)).astype(F)
    q[-C // 8:] *= 40.0
    onew, oinfo = onuts.nuts_kernel(keys, ohmc.init(q, otgt), otgt, eps_c, imm, depth, margins=margins)
    new, info = bj.nuts.build_kernel(max_tree_depth=depth)(tk(keys), bj.nuts.init(tf(q), tgt), tgt, tf(eps_c), tf(imm), depth)
    torch.cuda.synchronize()
    same = ((npy(info.num_integration_steps) == oinfo.num_integration_steps)
            & (npy(info.num_trajectory_expansions) == oinfo.num_trajectory_expansions)
            & (npy(info.is_turning) == oinfo.is_turning) & (npy(info.is_divergent) == oinfo.is_divergent)
            & np.all(np.isclose(npy(new.position), onew.position, rtol=2e-3, atol=2e-4), axis=1))
    print(f"{metric}/{target} D={D}: {same.mean():.3f} identical; margins of the others {np.sort(margins[~same])[:6]}; tree sizes "
          f"{np.bincount(oinfo.num_integration_steps).nonzero()[0]}; divergent {int(oinfo.is_divergent.sum())}, "
          f"turning {int(oinfo.is_turning.sum())}, depths {np.bincount(oinfo.num_trajectory_expansions)}")
    assert len(np.unique(oinfo.num_integration_steps)) >= 3 and oinfo.is_divergent.any()   # the case does exercise the tree
    assert same.mean() >= 0.9
    assert (margins[~same] < 2e-3).all(), np.sort(margins[~same])[-3:]
    ok = same
    close_elementwise(npy(info.acceptance_rate)[ok], oinfo.acceptance_rate[ok], 2e-3, 1e-2)
    close_elementwise(npy(info.energy)[ok], oinfo.energy[ok], 1e-4, 1.0)
    close_elementwise(npy(new.logdensity)[ok], onew.logdensity[ok], 2e-4, 1.0)


# ---------------------------------------------------------------------------------------------------------------------
# per-chain dense metrics and per-chain dense Welford (what jax.vmap(window_adaptation(..., is_mass_matrix_diagonal=False)
# .run) carries: mass_matrix.py:411-442 outer-product update, metrics.py:712-715 factorisation per chain)
# ---------------------------------------------------------------------------------------------------------------------
from test_gpu_parity import close  # noqa: E402


def _spd_stack(rs, C, D, scale=1.0):
    A = rs.standard_normal((C, D, D))
    return (scale * (A @ A.transpose(0, 2, 1) / D + np.eye(D))).astype(F)


@pytest.mark.parametrize("kind, D", [("diag", 6), ("funnel", 20), ("diag", 64), ("banana", 2)])
def test_per_chain_dense_metric_matches_oracle(kind, D):
    from test_gpu_parity import make_target
    rs = np.random.default_rng(31 + D)
    tgt, otgt = make_target(kind, D, rs)
    C = 12
    imm = _spd_stack(rs, C, D)
    q = (0.4 * rs.standard_normal((C, D))).astype(F)
    keys = oprng.split(oprng.key(5), C)
    eng = _engine.Engine(DEV, C, D, tgt)
    eng.set_metric(tf(imm))
    # momentum draw p = L_c^-T z and velocity / energy with every chain's own matrix
    p_dev = npy(eng.sample_momentum(tk(keys)))
    p_ref = np.concatenate([ohmc.Metric(imm[c]).sample_momentum(keys[c:c + 1], D) for c in range(C)])
    close(p_dev, p_ref, rtol=1e-5)
    lp, _ = otgt(q)
    e_dev = npy(eng.energy(tf(p_ref), tf(lp)))
    e_ref = np.concatenate([-lp[c:c + 1] + ohmc.Metric(imm[c]).kinetic_energy(p_ref[c:c + 1]) for c in range(C)])
    close(e_dev, e_ref, rtol=1e-5, scale=np.max(np.abs(e_ref)) + 1)
    # HMC and NUTS transitions, teacher-forced, chain by chain through the oracle
    st = bj.hmc.init(tf(q), tgt)
    new, info = bj.hmc.build_kernel(full_info=True)(tk(keys), st, tgt, 0.1, tf(imm), 6)
    nnew, ninfo = bj.nuts.build_kernel(full_info=True)(tk(keys), st, tgt, 0.15, tf(imm), 6)
    torch.cuda.synchronize()
    for c in range(C):
        ost = ohmc.init(q[c:c + 1], otgt)
        onew, oinfo = ohmc.hmc_kernel(keys[c:c + 1], ost, otgt, F(0.1), imm[c], 6)
        close(npy(info.proposal.position)[c:c + 1], oinfo.proposal[0], rtol=2e-5)
        close(npy(info.energy)[c:c + 1], oinfo.energy, rtol=1e-5, scale=np.abs(oinfo.energy).max() + 1)
        if bool(npy(info.is_accepted)[c]) == bool(oinfo.is_accepted[0]):
            close(npy(new.position)[c:c + 1], onew.position, rtol=2e-5)
        o2, oi2 = onuts.nuts_kernel(keys[c:c + 1], ost, otgt, F(0.15), imm[c], 6)
        if int(npy(ninfo.num_integration_steps)[c]) == int(oi2.num_integration_steps[0]):
            assert np.allclose(npy(nnew.position)[c:c + 1], o2.position, rtol=1e-4, atol=1e-5) or \
                abs(float(npy(ninfo.acceptance_rate)[c]) - float(oi2.acceptance_rate[0])) < 1e-4
    n_same = sum(int(npy(ninfo.num_integration_steps)[c]) ==
                 int(onuts.nuts_kernel(keys[c:c + 1], ohmc.init(q[c:c + 1], otgt), otgt, F(0.15), imm[c], 6)[1]
                     .num_integration_steps[0]) for c in range(C))
    assert n_same >= C - 1
    with pytest.raises(bj.BjxError, match="dim <= 64"):
        e2 = _engine.Engine(DEV, 3, 100, T.StdNormal(100))
        e2.set_metric(torch.eye(100, device=DEV).repeat(3, 1, 1).contiguous())


def test_per_chain_dense_factorisation_non_pd_stays_in_its_chain():
    # L^-T per chain on the device (float64): a matrix that is not positive definite gives NaN momenta for ITS chain only
    # (jnp.linalg.cholesky semantics); the other chains match the oracle's factorisation
    C, D = 9, 48
    rs = np.random.default_rng(2)
    imm = _spd_stack(rs, C, D, scale=3.0)
    imm[4] = -imm[4]
    eng = _engine.Engine(DEV, C, D, T.StdNormal(D))
    eng.set_metric(tf(imm))
    keys = oprng.split(oprng.key(1), C)
    p = npy(eng.sample_momentum(tk(keys)))
    assert np.isnan(p[4]).any()
    for c in range(C):
        if c != 4:
            close(p[c:c + 1], ohmc.Metric(imm[c]).sample_momentum(keys[c:c + 1], D), rtol=1e-5)


def test_welford_dense_per_chain_kernels():
    from blackjax_b200._lib import check, lib, ptr
    C, D = 7, 10
    rs = np.random.default_rng(8)
    eng = _engine.Engine(DEV, C, D, T.StdNormal(D))
    mean = torch.zeros(C, D, device=DEV)
    m2 = torch.zeros(C, D, D, device=DEV)
    ws = [oadapt.welford_init(D, diagonal=False) for _ in range(C)]
    for n in range(1, 12):
        x = (rs.standard_normal((C, D)) * np.linspace(0.5, 3, D) + 1.0).astype(F)
        dx = tf(x)
        check(lib().bjx_welford_dense_update(eng.h, ptr(dx), ptr(mean), ptr(m2), n), eng.h)
        ws = [oadapt.welford_update(w, xi) for w, xi in zip(ws, x)]
    close(npy(mean), np.stack([w.mean for w in ws]), rtol=1e-5)
    close(npy(m2), np.stack([w.m2 for w in ws]), rtol=1e-5, scale=np.max([np.abs(w.m2).max() for w in ws]))
    imm = torch.empty(C, D, D, device=DEV)
    check(lib().bjx_welford_dense_final(eng.h, ptr(mean), ptr(m2), 11, ptr(imm)), eng.h)
    ref = np.stack([oadapt.welford_final(w) for w in ws])
    close(npy(imm), ref, rtol=1e-5, scale=np.abs(ref).max())
    assert float(mean.abs().max()) == 0.0 and float(m2.abs().max()) == 0.0


def test_window_adaptation_per_chain_dense_recovers_each_chains_covariance():
    """window_adaptation(nuts, target, is_mass_matrix_diagonal=False) with per-chain state (shared=False): every chain
    ends with its own dense inverse mass matrix [C, D, D] and step size; on a correlated Gaussian the matrices must
    approach the target covariance (Stan's regularisation and ~200 draws leave ~25 % element noise) and the adapted sampler
    must run with them."""
    D, C = 4, 64
    rs = np.random.default_rng(0)
    A = rs.standard_normal((D, D))
    cov = A @ A.T / D + 0.5 * np.eye(D)
    tgt = T.DenseGaussian(np.linalg.inv(cov))
    q0 = tf(rs.standard_normal((C, D)))
    warmup = bj.window_adaptation(bj.nuts, tgt, is_mass_matrix_diagonal=False)
    (state, params), _ = warmup.run(bj.random.key(3, DEV), q0, 400)
    imm = npy(params["inverse_mass_matrix"])
    assert imm.shape == (C, D, D) and npy(params["step_size"]).shape == (C,)
    assert np.all(np.isfinite(imm))
    mean_imm = imm.mean(0)
    assert np.max(np.abs(mean_imm - cov)) < 0.12 * np.max(np.abs(cov))       # averaged over chains: close to Sigma
    assert np.all(np.linalg.eigvalsh(imm.astype(np.float64)) > 0)            # every chain's matrix is SPD
    alg = bj.nuts(tgt, **params)
    st, acc = state, []
    for k in bj.random.split(bj.random.key(4, DEV), 30):
        st, info = alg.step(k, st)
        acc.append(float(info.acceptance_rate.mean()))
    assert 0.6 < np.mean(acc) < 0.98
