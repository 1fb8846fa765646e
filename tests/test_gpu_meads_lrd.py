"""GPU tests of MEADS-LRD (meads_adaptation(..., low_rank_rank=k)): the on-device eigensolver of bjx_meads_lrd_update /
bjx_meads_lrd_metric against float64 numpy.linalg.eigh, one warm-up step's statistics teacher-forced against
oracle/meads_lrd.py, and the reference's low-rank MEADS tests (tests/adaptation/test_meads.py
TestMEADSLowRank, TestMEADSLowRankHighDimFixes, TestMEADSLRDX64Sanity) replayed on the device."""
import warnings

import numpy as np
import pytest
import torch

import blackjax_b200 as bj
from blackjax_b200 import _engine, targets as T
from blackjax_b200.adaptation import meads_adaptation as mm
from blackjax_b200.mcmc.metrics import LowRankMetric
from oracle import meads_lrd as olrd

pytestmark = pytest.mark.gpu
F = np.float32
DEV = "cuda:0"


def tf(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(DEV)


def npy(t):
    return t.detach().cpu().numpy()


# ---- a Gaussian with precision I + V diag(c) V^T (V [D, r] orthonormal): O(D r) per gradient ------------------------
LOWRANK_GAUSSIAN = r"""
#pragma once
namespace bjx_user {
// theta = [r, c_0 .. c_{r-1}, V (D x r, row-major)];  logp = -1/2 (|x|^2 + sum_j c_j (V_j . x)^2)
template <class R>
struct Model {
  __device__ __forceinline__ void init(const bjx::UserCtx&) {}
  template <bool WANT_LOGP>
  __device__ __forceinline__ void value_and_grad(const bjx::UserCtx& u, const float (&q)[R::NS], float (&g)[R::NS],
                                                 float& logp) const {
    const int r = (int)u.theta[0];
    const float* c = u.theta + 1;
    const float* V = c + r;
    float quad = 0.f;
#pragma unroll
    for (int s = 0; s < R::NS; ++s) { g[s] = -q[s]; quad = fmaf(q[s], q[s], quad); }
    quad = bjx::warp_sum(quad);
    for (int j = 0; j < r; ++j) {
      float t = 0.f;
#pragma unroll
      for (int s = 0; s < R::NS; ++s) {
        const int e = R::idx(s, u.lane);
        if (e < u.D) t = fmaf(V[e * r + j], q[s], t);
      }
      t = bjx::warp_sum(t);
      quad = fmaf(c[j] * t, t, quad);
#pragma unroll
      for (int s = 0; s < R::NS; ++s) {
        const int e = R::idx(s, u.lane);
        if (e < u.D) g[s] = fmaf(-c[j] * t, V[e * r + j], g[s]);
      }
    }
    if (WANT_LOGP) logp = -0.5f * quad;
  }
};
}  // namespace bjx_user
"""


def lowrank_gaussian(D, r, c=99.0, seed=5):
    """precision I + V diag(c) V^T, c a number or [r]; returns (target, V)"""
    V, _ = np.linalg.qr(np.random.default_rng(seed).standard_normal((D, r)))
    theta = np.concatenate([[r], np.broadcast_to(c, (r,)), V.reshape(-1)]).astype(F)
    return T.UserTarget(D, LOWRANK_GAUSSIAN, theta, name=f"lrd_gauss_{D}_{r}"), V


# ---- eigensolver ----------------------------------------------------------------------------------------------------
def exact_samples(cov, C, offset=3.0, seed=0):
    """C rows whose float64 sample covariance is exactly `cov` (centred orthonormal columns times chol(cov)^T)."""
    D = cov.shape[0]
    z = np.random.default_rng(seed).standard_normal((C, D))
    q, _ = np.linalg.qr(z - z.mean(0))
    return (np.sqrt(C - 1) * q @ np.linalg.cholesky(cov).T + offset).astype(F)


def device_metric(x, k):
    """Fold x into a fresh accumulator (one in-window step) and return (bjx_meads_lrd_metric, header)."""
    C, D = x.shape
    q = tf(x)
    eng = _engine.get_engine(q, T.StdNormal(D))
    lr = mm._LowRank(eng, k, 1)
    lr.install()
    folds = mm._Folds(eng, 1)
    lr.update(folds, q, -q, 0, True, 0.5, 1.0)
    m = lr.metric(q)
    return tuple(npy(a).astype(np.float64) for a in m), npy(lr.header)


def planted_spectrum(D, k, seed, cluster=None, ratio=0.85):
    """Eigenvalues 1 + mu of a correlation matrix, mean exactly 1.  The top min(D, k + 4) |mu| fall geometrically (by
    `ratio`, signs alternating), so the gap at k is about 18 % by default; the bulk lies within about 0.02 of 1.  cluster = "same" /
    "mixed": the five scores at positions k - 2 .. k + 2 (1-based) are made exactly equal, with one sign or alternating
    signs, so the cluster straddles k."""
    rng = np.random.default_rng(seed)
    top = min(D, k + 4)
    s = 0.9 * ratio ** np.arange(top)
    sign = np.where(np.arange(top) % 2 == 0, 1.0, -1.0)
    if cluster is not None:
        lo = max(0, k - 3)
        s[lo:lo + 5] = s[min(lo + 2, top - 1)]
        if cluster == "same":
            sign[lo:lo + 5] = 1.0
    mu = np.zeros(D)
    mu[:top] = sign * s
    if D > top:
        mu[top:] = rng.uniform(-0.01, 0.01, D - top)
        mu[top:] -= mu.sum() / (D - top)
    return 1.0 + mu


def planted_cov(D, k, seed, cluster=None, ratio=0.85):
    """diag(sigma) R diag(sigma) with R = Q diag(lam) Q^T.  For D a power of two Q is a signed, permuted Sylvester
    Hadamard matrix / sqrt(D): every diagonal entry of R is then mean(lam) = 1, so R is exactly the correlation matrix
    and its spectrum is the planted one.  Otherwise Q is random and the normalisation moves the spectrum slightly."""
    rng = np.random.default_rng(seed)
    lam = planted_spectrum(D, k, seed, cluster, ratio)
    if D & (D - 1) == 0:
        from scipy.linalg import hadamard
        Q = hadamard(D)[rng.permutation(D)] * rng.choice([-1.0, 1.0], D) / np.sqrt(D)
    else:
        Q, _ = np.linalg.qr(rng.standard_normal((D, D)))
    R = (Q * lam) @ Q.T
    sigma = np.exp(rng.uniform(-1.0, 1.0, D))
    return sigma[:, None] * R * sigma[None, :]


def reference(x, k):
    """float64 (sigma, A = R - I, eigenvalues and eigenvectors of R by |lam - 1| descending) of x's sample covariance."""
    cov = np.cov(x.astype(np.float64), rowvar=False)
    sigma = np.sqrt(np.diag(cov))
    R = cov / sigma[:, None] / sigma[None, :]
    lam, V = np.linalg.eigh(R)
    order = np.argsort(np.abs(lam - 1.0), kind="stable")[::-1]
    return sigma, R - np.eye(len(sigma)), lam[order], V[:, order]


def check_pairs(A, U, lam, nrm):
    """residuals ||A u - mu u|| <= 1e-4 ||A||, ||U^T U - I||_max <= 1e-5, |mu| descending"""
    mu = lam - 1.0
    assert np.all(np.diff(np.abs(mu)) <= 0), mu
    res = np.linalg.norm(A @ U - U * mu, axis=0)
    assert np.max(res) <= 1e-4 * nrm, res
    assert np.max(np.abs(U.T @ U - np.eye(U.shape[1]))) <= 1e-5


EIG_CASES = [(6, 1), (6, 3), (40, 3), (40, 10), (40, 16), (256, 1), (256, 10), (256, 16), (512, 3), (512, 16)]


@pytest.mark.parametrize("D,k", EIG_CASES)
def test_eigensolver_matches_float64_eigh(D, k):
    x = exact_samples(planted_cov(D, k, seed=D + k), 4096)
    (sigma, U, lam), hdr = device_metric(x, k)
    s0, A, lam0, V0 = reference(x, k)
    nrm = np.max(np.abs(lam0 - 1.0))
    assert hdr[mm._LowRank.ENGAGED] == 1 and hdr[mm._LowRank.NOCONV] == 0, hdr[:8]
    assert np.max(np.abs(sigma / s0 - 1.0)) <= 1e-6
    assert np.max(np.abs(lam - lam0[:k])) <= 2e-5 * nrm
    check_pairs(A, U, lam, nrm)
    gaps = np.abs(lam0 - 1.0)
    if k < D:                                    # the planted spectra have a gap of >= 10 % at k (asserted)
        assert gaps[k - 1] >= 1.1 * gaps[k], (gaps[k - 1], gaps[k])
        U0 = V0[:, :k]
        assert np.linalg.norm(U @ U.T - U0 @ U0.T) <= 1e-4
        M = olrd.dense_inverse_mass(sigma, U, lam)
        M0 = olrd.dense_inverse_mass(s0, U0, lam0[:k])
        assert np.max(np.abs(M - M0)) <= 1e-4 * np.max(np.abs(M0))


@pytest.mark.parametrize("D,k,kind", [(64, 3, "same"), (256, 10, "same"), (256, 10, "mixed")])
def test_eigensolver_cluster_straddling_k(D, k, kind):
    """Five exactly equal |lam - 1| at positions k - 2 .. k + 2: any k-subset of the cluster's eigenspace is right, so
    the checks are the residuals, finiteness and the k-th |mu|."""
    x = exact_samples(planted_cov(D, k, seed=7, cluster=kind), 4096)
    (sigma, U, lam), hdr = device_metric(x, k)
    _, A, lam0, _ = reference(x, k)
    nrm = np.max(np.abs(lam0 - 1.0))
    sc = np.abs(lam0 - 1.0)
    assert np.ptp(sc[k - 3:k + 2]) <= 1e-5 * nrm and sc[k + 2] < 0.9 * sc[k - 1]   # the planted cluster is there
    assert hdr[mm._LowRank.NOCONV] == 0, hdr[:8]
    assert np.isfinite(U).all() and np.isfinite(lam).all()
    check_pairs(A, U, lam, nrm)
    assert abs(abs(lam[k - 1] - 1.0) - sc[k - 1]) <= 1e-4 * nrm


def test_eigensolver_collinear_input_is_floored():
    C, D, k = 4096, 40, 3
    z = np.random.default_rng(2).standard_normal((C, 1))
    x = (z * np.linspace(0.5, 2.0, D)[None, :] + 1.0).astype(F)
    (sigma, U, lam), _ = device_metric(x, k)
    assert np.isfinite(sigma).all() and np.isfinite(U).all() and np.isfinite(lam).all()
    assert np.all(lam >= np.float32(1e-6))
    assert abs(lam[0] - D) <= 1e-3 * D


# ---- one warm-up step teacher-forced against the oracle ------------------------------------------------------------
def _planted_target(D, k):
    """A Gaussian whose correlation spectrum is planted as in planted_spectrum (top k + 4 scores with ~18 % gaps) and
    the exact-covariance ensemble that starts in it: a DenseGaussian at D <= 128, else the low-rank-precision user
    target with cov = I + V diag(mu) V^T (c = 1 / (1 + mu) - 1).  At D = 40, k = 3 the scores fall by 0.7 per step, so
    the gap at k stays open under the window's sampling noise."""
    if D <= 128:
        cov = planted_cov(D, k, seed=11, ratio=0.7 if k == 3 else 0.85)
        return T.DenseGaussian(np.linalg.inv(cov).astype(F)), cov
    r = k + 4
    mu = planted_spectrum(r, r, seed=11)[:r] - 1.0
    tgt, V = lowrank_gaussian(D, r, c=1.0 / (1.0 + mu) - 1.0, seed=12)
    return tgt, np.eye(D) + (V * mu) @ V.T


@pytest.mark.parametrize("D,k", [(40, 3), (40, 16), (256, 3), (256, 16)])
def test_teacher_forced_statistics_match_oracle(D, k):
    """40 steps, window from step 20: both sides see the same positions each step.  Every engaged step checks the
    device metric's eigenvalues (2e-5 ||A||), residuals (1e-4 ||A||) and orthonormality (1e-5) against the oracle's
    accumulator; where the accumulated spectrum has a gap of >= 10 % at k, also the implied dense M^-1 (1e-4)."""
    C, K, steps, frac = 4096, 4, 40, 0.5
    tgt, cov = _planted_target(D, k)
    q0 = exact_samples(cov, C, offset=0.0, seed=D + k)
    q = tf(q0)
    eng = mm._engine_for(q, tgt)
    st = bj.ghmc.init(q.clone(), tgt, bj.random.key(1, DEV))
    folds, diag = mm._Folds(eng, K), mm._Folds(eng, K)
    lr = mm._LowRank(eng, k, K)
    lr.install()
    kernel = bj.ghmc.build_kernel(inplace=True)
    keys = bj.random.split(bj.random.key(2, DEV), steps)
    acc = olrd.moment_block_init(D)
    start = int(frac * steps)
    n = C // K
    gated = 0
    for t in range(steps):
        x, g = npy(st.position), npy(st.logdensity_grad)
        diag.update(st.position, st.logdensity_grad, t, 0.5, 1.0)
        lr.update(folds, st.position, st.logdensity_grad, t, t >= start, 0.5, 1.0)
        acc, on, s_o, U_o, lam_o = olrd.step_metric(acc, x, k, t >= start)
        hdr = npy(lr.header)
        assert bool(hdr[lr.ENGAGED]) == on and hdr[lr.NOCONV] == 0, (t, hdr[:8])
        assert torch.equal(folds.step_size, diag.step_size) and torch.equal(folds.sigma, diag.sigma)
        sigma, U, lam = (npy(a).astype(np.float64) for a in (lr.sigma, lr.U, lr.lam))
        if on:
            np.testing.assert_allclose(sigma, s_o, rtol=1e-5)
            c64 = acc.m2.astype(np.float64) / (float(acc.count) - 1.0)
            s64 = np.sqrt(np.diag(c64))
            A = c64 / np.outer(s64, s64) - np.eye(D)
            ev = np.linalg.eigvalsh(A)
            nrm = np.max(np.abs(ev))
            assert np.max(np.abs(lam - lam_o)) <= 2e-5 * nrm, t
            check_pairs(A, U, lam, nrm)
            gaps = np.sort(np.abs(ev))[::-1]
            if gaps[k - 1] >= 1.1 * gaps[k]:
                gated += 1
                M, M0 = olrd.dense_inverse_mass(sigma, U, lam), olrd.dense_inverse_mass(s_o, U_o, lam_o)
                assert np.max(np.abs(M - M0)) <= 1e-4 * np.max(np.abs(M0)), t
        else:
            np.testing.assert_allclose(sigma, s_o, rtol=2e-6)   # pooled from the fold moments: not bit-identical
            assert np.array_equal(U, U_o) and np.array_equal(lam, lam_o)
        _, _, al_o, de_o = olrd.fold_parameters(x, g, t, K, sigma.astype(F), U.astype(F), lam.astype(F))
        np.testing.assert_allclose(npy(folds.alpha), al_o, rtol=1e-4)
        np.testing.assert_allclose(npy(folds.delta), de_o, rtol=1e-4)
        skip = ((t % K) * n, (t % K + 1) * n)
        st, _ = kernel(keys[t], st, tgt, None, None, None, None,
                       _rows=(folds.step_size, folds.alpha, folds.delta, None, None, n, skip))
    print(f"D={D} k={k}: dense M^-1 checked on {gated} of {steps - start} engaged steps")
    if (D, k) == (40, 3):
        assert gated > 0


# ---- the reference's low-rank MEADS tests, on the device ------------------------------------------------------------
def _run(tgt, x0, key=0, steps=20, **kw):
    algo = bj.meads_adaptation(tgt, x0.shape[0], **kw)
    (state, params), _ = algo.run(bj.random.key(key, DEV), tf(x0), steps)
    return state, params


def _corr_target(D=6, rho=0.9):
    """make_correlated_pair_logdensity (test_meads.py:257-271): dims 0 and 1 correlated by rho"""
    cov = np.eye(D)
    cov[0, 1] = cov[1, 0] = rho
    return T.DenseGaussian(np.linalg.inv(cov).astype(F))


def _finite_metric(m):
    return all(np.isfinite(npy(a)).all() for a in m)


def test_none_rank_is_identical_to_default():
    x0 = np.random.default_rng(0).standard_normal((64, 6)).astype(F)
    a_state, a = _run(_corr_target(), x0, num_folds=4)
    b_state, b = _run(_corr_target(), x0, num_folds=4, low_rank_rank=None)
    for name in a:
        assert torch.equal(a[name], b[name]), name
    assert torch.equal(a_state.position, b_state.position)


def test_shapes_orthonormality_and_clamps():
    """TestMEADSLowRank shapes and test_low_rank_rank_clamped_to_dimension (C = 32, K = 4, D = 6, k = 7 -> 6)."""
    x0 = np.random.default_rng(1).standard_normal((32, 6)).astype(F)
    _, p = _run(_corr_target(), x0, num_folds=4, low_rank_rank=2)
    m = p["momentum_inverse_scale"]
    assert isinstance(m, LowRankMetric)
    assert m.sigma.shape == (6,) and m.U.shape == (6, 2) and m.lam.shape == (2,)
    U = npy(m.U).astype(np.float64)
    assert np.max(np.abs(U.T @ U - np.eye(2))) <= 1e-4
    state, p = _run(_corr_target(), x0, num_folds=4, low_rank_rank=7)     # clamped to D
    assert p["momentum_inverse_scale"].U.shape == (6, 6) and torch.isfinite(state.position).all()
    x3 = np.random.default_rng(2).standard_normal((4, 6)).astype(F)
    _, p = _run(_corr_target(), x3, num_folds=1, low_rank_rank=5)           # clamped to num_chains - 1
    assert p["momentum_inverse_scale"].U.shape == (6, 3)


def test_argument_errors():
    with pytest.raises(ValueError, match="low_rank_rank"):
        bj.meads_adaptation(_corr_target(), 1, num_folds=1, low_rank_rank=2)
    with pytest.raises(ValueError):
        bj.meads_adaptation(_corr_target(), 8, num_folds=1, low_rank_rank=2, low_rank_window_fraction=1.5)
    x0 = np.random.default_rng(0).standard_normal((64, 200)).astype(F)
    prec = np.eye(200, dtype=F)
    with pytest.raises(NotImplementedError):                               # dense route: no low-rank metric
        _run(T.DenseGaussian(prec), x0, num_folds=4, low_rank_rank=2, steps=1)


def test_first_step_size_matches_diagonal_run():
    """test_step_size_independent_of_low_rank_metric: C = 16, K = 4, D = 6, k = 3, one step."""
    x0 = np.random.default_rng(3).standard_normal((16, 6)).astype(F)
    _, a = _run(_corr_target(), x0, steps=1, num_folds=4)
    _, b = _run(_corr_target(), x0, steps=1, num_folds=4, low_rank_rank=3)
    assert torch.equal(a["step_size"], b["step_size"])


def test_collinear_initial_ensemble_is_floored():
    """test_low_rank_floors_degenerate_eigenvalues_collinear_init: C = 32, K = 4, D = 6, k = 3, 20 steps."""
    rng = np.random.default_rng(4)
    direction = rng.standard_normal(6)
    direction /= np.linalg.norm(direction)
    x0 = (rng.standard_normal((32, 1)) * direction[None, :]).astype(F)
    state, p = _run(_corr_target(), x0, steps=20, num_folds=4, low_rank_rank=3)
    m = p["momentum_inverse_scale"]
    assert (npy(m.lam) >= np.float32(1e-6)).all() and np.isfinite(npy(m.lam)).all()
    assert torch.isfinite(state.position).all()


def test_higher_dim_no_step_size_collapse():
    """test_low_rank_higher_dim_no_step_size_collapse: C = 32, K = 4, D = 40, precision I + 24 d d^T, k = 10, 60 steps."""
    D, C = 40, 32
    d = np.random.default_rng(0).standard_normal(D)
    d /= np.linalg.norm(d)
    tgt = T.DenseGaussian((np.eye(D) + 24.0 * np.outer(d, d)).astype(F))
    x0 = np.random.default_rng(5).standard_normal((C, D)).astype(F)
    state, p = _run(tgt, x0, steps=60, num_folds=4, low_rank_rank=10)
    assert float(p["step_size"]) > 1e-2
    assert torch.isfinite(state.position).all() and np.isfinite(npy(p["momentum_inverse_scale"].lam)).all()


def test_captures_correlated_subspace_and_draws_are_finite():
    """test_low_rank_metric_captures_correlated_subspace: C = 32, K = 4, D = 6, k = 2, 40 steps; then draws from
    blackjax.ghmc(target, **params) stay finite."""
    tgt = _corr_target()
    x0 = np.random.default_rng(42).standard_normal((32, 6)).astype(F)
    _, p = _run(tgt, x0, key=42, steps=40, num_folds=4, low_rank_rank=2)
    U = npy(p["momentum_inverse_scale"].U).astype(np.float64)
    assert np.sqrt(U[0, 0] ** 2 + U[1, 0] ** 2) > 0.5
    sampler = bj.ghmc(tgt, **dict(p))
    state = sampler.init(tf(x0), bj.random.key(9, DEV))
    for i in range(10):
        state, _ = sampler.step(bj.random.key(10 + i, DEV), state)
    assert torch.isfinite(state.position).all()


def test_run_sanity():
    """TestMEADSLRDX64Sanity's bounds (in float32): D = 6, C = 16, K = 4, k = 3, 20 steps."""
    x0 = np.random.default_rng(6).standard_normal((16, 6)).astype(F)
    with warnings.catch_warnings():
        warnings.simplefilter("error", RuntimeWarning)             # every eigensolve converged
        state, p = _run(_corr_target(), x0, steps=20, num_folds=4, low_rank_rank=3)
    m = p["momentum_inverse_scale"]
    assert float(p["step_size"]) > 0.0
    assert np.isfinite(npy(m.lam)).all() and (npy(m.lam) >= np.float32(1e-6)).all()
    assert torch.isfinite(state.position).all() and _finite_metric(m)


def test_recovers_planted_subspace_and_is_deterministic():
    D, r, C = 256, 4, 4096
    tgt, V = lowrank_gaussian(D, r)
    x0 = np.random.default_rng(6).standard_normal((C, D)).astype(F)
    s1, p1 = _run(tgt, x0, key=3, steps=60, num_folds=4, low_rank_rank=r)
    U = npy(p1["momentum_inverse_scale"].U).astype(np.float64)
    cosines = np.linalg.svd(V.T @ U, compute_uv=False)
    assert cosines.min() > 0.9, cosines
    s2, p2 = _run(tgt, x0, key=3, steps=60, num_folds=4, low_rank_rank=r)
    assert torch.equal(s1.position, s2.position)
    for a, b in zip(p1["momentum_inverse_scale"], p2["momentum_inverse_scale"]):
        assert torch.equal(a, b)
