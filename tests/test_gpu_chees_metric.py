"""GPU tests of ChEES with mass_matrix_estimation="diagonal": the SYRK covariance accumulator against float64 numpy, the
device update teacher-forced against oracle/chees.py, bit-identity with the identity path when the
window never opens, the statistics of a warm-up on a target a diagonal metric cannot whiten, and independence of the GPU
count."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import blackjax_b200 as bj
from blackjax_b200 import _engine, targets as T
from blackjax_b200._lib import CHEES_LENGTH_FLOOR, CHEES_WHITEN, check, lib, ptr
from blackjax_b200.adaptation.chees_adaptation import adam
from oracle import adaptation as oadapt
from oracle import chees as ochees
from oracle import prng as oprng
from oracle import targets as otargets

pytestmark = pytest.mark.gpu
F = np.float32
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPTS = CHEES_WHITEN | CHEES_LENGTH_FLOOR


def tf(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(DEV)


def npy(t):
    return t.detach().cpu().numpy()


@pytest.mark.parametrize("D", [1, 3, 24, 100, 132, 512, 1024])
@pytest.mark.parametrize("C", [1, 37, 4096, 4609])
def test_syrk_covariance_accumulator_vs_float64(C, D):
    """Three folds of shifted, correlated snapshots into the per-block accumulators (bjx_chees_metric_fold_covariance),
    merged (bjx_chees_metric_covariance): count, mean and covariance against float64 numpy, the covariance within 1e-5 of
    its largest diagonal entry.  The dimensions cover a partial 64-wide tile below and above 128 (handles take dim <= 128
    or dim % 4 == 0), one and several tiles, and the 1024 limit; the chain counts one chain, a partial 16-row chunk, one
    full block and a ragged second block."""
    rng = np.random.default_rng(C * 7 + D)
    A = rng.standard_normal((D, D)) / math.sqrt(D) + np.eye(D)
    xs = [(rng.standard_normal((C, D)) @ A.T * np.logspace(-0.5, 0.5, D) + 2.0 + k).astype(F) for k in range(3)]
    q0 = tf(xs[0])
    eng = _engine.get_engine(q0, T.DiagGaussian(np.ones(D)))
    L_ = lib()
    ms = torch.empty(L_.bjx_chees_metric_state_floats(C, D, 1, OPTS), device=DEV)
    imm = torch.empty(D, device=DEV)
    check(L_.bjx_chees_metric_init(eng.h, ptr(ms), 1, OPTS, ptr(imm)), eng.h)
    for x in xs:
        check(L_.bjx_chees_metric_fold_covariance(eng.h, OPTS, ptr(ms), ptr(tf(x))), eng.h)
    out = torch.empty(1 + D + D * D, device=DEV)
    check(L_.bjx_chees_metric_covariance(eng.h, None, 1, OPTS, ptr(ms), ptr(out)), eng.h)
    o = npy(out)
    allx = np.concatenate(xs).astype(np.float64)
    ref = np.atleast_2d(np.cov(allx, rowvar=False))
    assert o[0] == 3 * C
    np.testing.assert_allclose(o[1:1 + D], allx.mean(0), rtol=1e-5, atol=1e-5)
    cov = o[1 + D:].reshape(D, D)
    err = np.max(np.abs(cov - ref)) / np.max(np.diag(ref))
    assert err <= 1e-5, err
    assert np.array_equal(cov, cov.T)


@pytest.mark.parametrize("D", [24, 200])
def test_chees_update_metric_teacher_forced_vs_oracle(D):
    """Every step the device update (bjx_chees_update_metric) and the oracle are fed the SAME transition; window from step
    50 of 100 (recomputes at 64 and 96), 4608 chains (a ragged second block).  Per step: step size and trajectory length
    within 1e-5, imm within 1e-5 of float64 moments, the engagement flag exactly, lambda_max within 1e-4, and the step count exactly unless
    jitter * T / eps is within rounding of an integer."""
    C, T_, start = 4608, 100, 50
    scale = np.logspace(-0.5, 1.0, D)
    tgt = T.DiagGaussian(scale)
    q = (np.random.default_rng(2).standard_normal((C, D)) * scale).astype(F)
    kernel = bj.hmc.build_kernel(full_info=True)
    state = bj.hmc.init(tf(q), tgt)
    eng = _engine.get_engine(state.position, tgt)
    L_ = lib()
    max_bits = 11
    st = torch.empty(L_.bjx_chees_state_floats(C, D, 1), device=DEV)
    ms = torch.empty(L_.bjx_chees_metric_state_floats(C, D, 1, OPTS), device=DEV)
    eps_c = torch.empty(C, device=DEV)
    steps_c = torch.empty(C, dtype=torch.int32, device=DEV)
    imm = torch.empty(D, device=DEV)
    lam = torch.zeros(T_, device=DEV)
    engd = torch.zeros(T_, device=DEV)
    check(L_.bjx_chees_init(eng.h, ptr(st), 0.05, max_bits, 1.0, ptr(eps_c), ptr(steps_c)), eng.h)
    check(L_.bjx_chees_metric_init(eng.h, ptr(ms), 1, OPTS, ptr(imm)), eng.h)
    eng._imm, eng._imm_key = imm, (imm.data_ptr(), tuple(imm.shape), imm._version, str(imm.device))
    os_ = ochees.chees_init(0.05)
    wf, cov, eig = oadapt.welford_init(D), oadapt.moment_block_init(D), ochees.eig_state_init(D)
    thresh = ochees.engagement_threshold(D)
    keys = bj.random.split(bj.random.key(5, DEV), T_)
    near_integer = 0
    n64, mean64, m2_64 = 0, np.zeros(D), np.zeros(D)
    for t in range(T_):
        imm_or = ochees.diagonal_imm(wf, thresh, D)
        imm_dev = npy(imm)
        # imm against the same window's float64 moments; the oracle's row-by-row float32 fold (up to 230k rows) drifts
        # from them by a few 1e-5, so it is held to 1e-4
        imm64 = np.maximum(m2_64 / (n64 - 1), 1e-20) if n64 >= thresh else np.ones(D)
        np.testing.assert_allclose(imm_dev, imm64, rtol=1e-5)
        np.testing.assert_allclose(imm_or, imm64, rtol=1e-4)
        consumed, _ = ochees.apply_length_floor(os_.trajectory_length, eig.lambda_max, wf.n >= thresh, True, 1000, os_.step_size)
        L_or = ochees.integration_steps(os_.random_generator_arg, F(consumed / os_.step_size), 1.0, max_bits)
        x = float(ochees.jitter(os_.random_generator_arg, 1.0, max_bits)) * float(consumed / os_.step_size)
        L_dev = int(steps_c[0])
        if L_dev != L_or:
            assert abs(x - round(x)) < 1e-4 * max(x, 1.0), (t, L_dev, L_or, x)
            near_integer += 1
        init_q = state.position
        state, info = kernel(keys[t], state, tgt, eps_c, imm, steps_c)
        in_window = t >= start
        recompute = in_window and t % 32 == 0
        check(L_.bjx_chees_update_metric(eng.h, None, 1, OPTS, ptr(st), ptr(ms), ptr(init_q), ptr(info.proposal.position),
                                         ptr(info.proposal.momentum), ptr(state.position), ptr(info.acceptance_rate),
                                         ptr(info.is_divergent.to(torch.uint8)), 0.1, 0.9, 0.999, 0.651, 0.5, 1000,
                                         int(in_window), int(recompute), ptr(eps_c), ptr(steps_c), None, ptr(imm), ptr(lam),
                                         ptr(engd)), eng.h)
        os_ = ochees.chees_update(os_, npy(info.proposal.position), npy(info.proposal.momentum), npy(init_q),
                                  npy(info.acceptance_rate), npy(info.is_divergent), imm=imm_dev, lr=0.1, max_bits=max_bits)
        newq = npy(state.position)
        if in_window:
            b64 = newq.astype(np.float64)
            mb = b64.mean(0)
            delta = mb - mean64
            n_ab = n64 + C
            m2_64 = m2_64 + ((b64 - mb) ** 2).sum(0) + delta * delta * (n64 * C / n_ab)
            mean64, n64 = mean64 + delta * (C / n_ab), n_ab
            wf = ochees.welford_fold(wf, newq)
            cov = oadapt.cgl_update_batch(cov, newq)
            if recompute:
                eig = ochees.recompute_eig(cov, imm_dev, eig)
        hdr = npy(st[:16])
        np.testing.assert_allclose(hdr[[0, 2]], [os_.step_size, os_.trajectory_length], rtol=1e-5)
        assert bool(npy(engd)[t]) == (wf.n >= thresh), t
        assert abs(float(npy(lam)[t]) - float(eig.lambda_max)) <= 1e-4 * float(eig.lambda_max), (t, npy(lam)[t], eig.lambda_max)
        # teacher forcing of the scalar state, as in the identity-metric test
        st[0], st[1], st[2], st[3] = float(os_.step_size), float(os_.log_step_size_ma), float(os_.trajectory_length), float(os_.log_trajectory_length_ma)
        st[4], st[5], st[7] = float(os_.da.log_step_size), float(os_.da.log_step_size_avg), float(os_.da.avg_error)
        st[10], st[11] = float(os_.optim.mu), float(os_.optim.nu)
    assert npy(engd)[start] == 1 and npy(engd)[start - 1] == 0
    assert npy(lam)[63] == 1.0 and npy(lam)[64] != 1.0
    assert near_integer <= 3


def test_window_fraction_one_bit_identical_to_identity_metric():
    """With the window never open the diagonal mode runs the identity metric: positions, per-step history (step sizes,
    trajectory lengths, step counts, gradients) and the final step size are bit-identical to mass_matrix_estimation=None."""
    C, D = 2048, 16
    tgt = T.DiagGaussian(np.logspace(-1, 1, D))
    q0 = bj.random.normal(bj.random.split(bj.random.key(3, DEV), C), (D,))
    warm0 = bj.chees_adaptation(tgt, num_chains=C)
    warm1 = bj.chees_adaptation(tgt, num_chains=C, mass_matrix_estimation="diagonal", mass_matrix_window_fraction=1.0)
    (l0, a), h0 = warm0.run(bj.random.key(9, DEV), q0.clone(), step_size=0.05, optim=adam(0.05), num_steps=60)
    (l1, b), info = warm1.run(bj.random.key(9, DEV), q0.clone(), step_size=0.05, optim=adam(0.05), num_steps=60)
    p0, p1, h1 = npy(l0.position), npy(l1.position), info.history
    assert np.array_equal(p0, p1)
    bits0, bits1 = h0.numpy().view(np.int32), h1.numpy().view(np.int32)   # bitwise: NaN gradients compare equal too
    assert np.array_equal(bits0, bits1), np.argwhere(bits0 != bits1)[:5]
    assert a["step_size"] == b["step_size"]
    assert torch.equal(b["inverse_mass_matrix"].cpu(), torch.ones(D))
    assert abs(b["integration_steps_params"][0] / a["integration_steps_params"][0] - 1) < 1e-5
    assert not info.engaged.any() and not info.floor_clipped_by_cap


def _slow_direction_target(D=64, seed=0):
    rng = np.random.default_rng(seed)
    u = rng.standard_normal(D)
    u /= np.linalg.norm(u)
    s = np.logspace(-1, 1, D)
    cov = (np.eye(D) + 24.0 * np.outer(u, u)) * s[:, None] * s[None, :]
    return cov


def test_chees_diagonal_statistics_slow_direction():
    """64-D Gaussian with scales logspace(-1, 1) and one slow direction (I + 24 u u^T) a diagonal metric cannot remove:
    imm within 10 % of diag(Sigma), lambda_max within 10 % of the top eigenvalue of the whitened Sigma, the adapted
    leapfrog count at or above the floor, step size / leapfrog count within 15 % / 30 % of the oracle's free run, and
    dynamic HMC with the adapted parameters recovering the marginal standard deviations within 15 %."""
    D, C, steps = 64, 1024, 300
    cov = _slow_direction_target(D)
    prec = np.linalg.inv(cov)
    tgt, otgt = T.DenseGaussian(prec), otargets.DenseGaussian(prec)
    q = (np.random.default_rng(1).standard_normal((C, D)) @ np.linalg.cholesky(cov).T).astype(F)
    warm = bj.chees_adaptation(tgt, num_chains=C, mass_matrix_estimation="diagonal")
    (last, params), info = warm.run(bj.random.key(21, DEV), tf(q), step_size=0.05, optim=adam(0.05), num_steps=steps)
    imm = npy(params["inverse_mass_matrix"])
    np.testing.assert_allclose(imm, np.diag(cov), rtol=0.10)
    sd = np.sqrt(np.diag(cov))
    top = np.linalg.eigvalsh(cov / sd[:, None] / sd[None, :])[-1]
    lam = float(info.lambda_max[-1])
    eps, n_lf = params["step_size"], params["integration_steps_params"][0]
    r = ochees.chees_run(otgt, oprng.key(21), q, 0.05, lr=0.05, num_steps=steps, mass_matrix_estimation="diagonal")
    print(f"device eps {eps:.4f} n_lf {n_lf:.2f} lambda {lam:.2f}; oracle eps {float(r.step_size):.4f} "
          f"n_lf {float(r.num_leapfrog_steps):.2f} lambda {float(r.lambda_max):.2f}; top eigenvalue {top:.2f}")
    assert abs(lam / top - 1) < 0.10
    assert n_lf >= (math.pi / 2) * math.sqrt(lam) / eps * (1 - 1e-5)
    assert abs(eps / float(r.step_size) - 1) < 0.15
    assert abs(n_lf / float(r.num_leapfrog_steps) - 1) < 0.30
    alg = bj.dhmc(tgt, **params)
    state = last
    draws = []
    for k in bj.random.split(bj.random.key(8, DEV), 200):
        state, _ = alg.step(k, state)
        draws.append(state.position)
    x = torch.stack(draws[50:]).reshape(-1, D)
    np.testing.assert_allclose(npy(x.std(0)), sd, rtol=0.15)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_chees_diagonal_bit_identical_on_one_and_two_gpus(tmp_path):
    worker = os.path.join(ROOT, "tests", "helpers", "chees_metric_worker.py")
    one, two = str(tmp_path / "g1.npz"), str(tmp_path / "g2.npz")
    env = dict(os.environ, PYTHONPATH=ROOT)
    subprocess.run([sys.executable, worker, one, "8192"], check=True, env=env, timeout=600)
    subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
                    "127.0.0.1", "--master-port", "29519", worker, two, "4096"], check=True, env=env, timeout=600)
    a, b = np.load(one), np.load(two)
    assert a["n_ranks"] == 1 and b["n_ranks"] == 2
    for k in ("history", "lambda_max", "engaged", "imm", "step_size", "n_lf", "position"):
        assert np.array_equal(a[k], b[k]), k
