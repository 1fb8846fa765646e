"""GPU tests of window_adaptation_low_rank: the device fold and window-end estimator teacher-forced against the float64
oracle (oracle/low_rank_window.py), the whole update loop teacher-forced under Stan's and the growing
schedule, the reference's statistical tests (tests/adaptation/test_low_rank_adaptation.py) pooled over chains, bit
identity and the rejections."""
import numpy as np
import pytest
import torch

import blackjax_b200 as bj
from blackjax_b200 import _engine, targets as T
from blackjax_b200._lib import BjxError
from blackjax_b200.adaptation import low_rank_adaptation as lra
from blackjax_b200.mcmc.metrics import LowRankMetric
from oracle import low_rank_window as o

pytestmark = pytest.mark.gpu
F = np.float32
DEV = "cuda:0"


def tf(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(DEV)


def npy(t):
    return t.detach().cpu().numpy().astype(np.float64)


# ---- a Gaussian with precision I + V diag(c) V^T (V [D, r] orthonormal) ---------------------------------------------
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


def rotated_gaussian(D, r=10, kappa=100.0, seed=5):
    """Covariance I - V diag(1 - v) V^T with v log-spaced from 1 / kappa to 1 (the mclmc_lrd recipe): returns (target, V,
    covariance)."""
    V, _ = np.linalg.qr(np.random.default_rng(seed).standard_normal((D, r)))
    v = np.logspace(-np.log10(kappa), 0.0, r, endpoint=False)
    c = 1.0 / v - 1.0
    theta = np.concatenate([[r], c, V.reshape(-1)]).astype(F)
    cov = np.eye(D) - (V * (1.0 - v)) @ V.T
    return T.UserTarget(D, LOWRANK_GAUSSIAN, theta, name=f"lrw_gauss_{D}_{r}"), V, cov


# ---- teacher forcing ------------------------------------------------------------------------------------------------
def planted(D, k, rows, seed, offset=0.7):
    """draws with k large-variance and k small-variance planted directions (gap >= 10 % at k in both the draws' and the
    scores' spectrum), and their exact Gaussian scores"""
    rs = np.random.default_rng(seed)
    Qm, _ = np.linalg.qr(rs.standard_normal((D, D)))
    var = np.ones(D) + rs.uniform(-0.02, 0.02, D)
    nk = min(k, D // 2)
    var[:nk] = np.geomspace(12.0, 3.0, nk) if nk > 1 else [12.0]
    var[nk:2 * nk] = np.geomspace(0.08, 0.3, nk) if nk > 1 else [0.08]
    scale = np.exp(rs.uniform(-0.5, 0.5, D))
    L = scale[:, None] * (Qm * np.sqrt(var))
    z = rs.standard_normal((rows, D))
    x = z @ L.T + offset
    prec = np.linalg.inv(L @ L.T)
    g = -(x - offset) @ prec + 0.05
    return x.astype(F), g.astype(F)


def window(eng, k, xs, gs, retained_from, gamma=1e-5, cutoff=2.0):
    """Run one slow window of len(xs) steps ([T, C, D]) through bjx_lowrank_window_update; returns the device state."""
    lw = lra._LowRankWindow(eng, k)
    lw.install(1.0)
    Tn, C, _ = xs.shape
    acc = torch.full((C,), 0.8, device=DEV)
    for t in range(Tn):
        b = 1 | (4 if t >= retained_from else 0) | (2 if t == Tn - 1 else 0)
        lw.update(tf(xs[t]), tf(gs[t]), acc, b, 0.8, gamma, cutoff)
    return lw


def compare_metric(lw, ref, k):
    _, mu, m = lw.final()
    sigma, U, lam = (npy(a) for a in m)
    s0, mu0, U0, lam0 = ref
    np.testing.assert_allclose(sigma, s0, rtol=1e-5)
    np.testing.assert_allclose(npy(mu), mu0, rtol=1e-5, atol=1e-5 * np.abs(mu0).max())
    M, M0 = o.implied_inverse_mass_matrix(sigma, U, lam), o.implied_inverse_mass_matrix(s0, U0, lam0)
    assert np.linalg.norm(M - M0) <= 1e-4 * np.linalg.norm(M0), np.linalg.norm(M - M0) / np.linalg.norm(M0)
    inf = lam != 1.0
    inf0 = lam0 != 1.0
    assert inf.sum() == inf0.sum(), (lam, lam0)
    np.testing.assert_allclose(np.sort(lam[inf]), np.sort(lam0[inf0]), rtol=1e-4)
    padded = np.all(U == 0.0, axis=0)
    assert np.all(lam[padded] == 1.0)
    Un = U[:, ~padded]
    assert np.max(np.abs(Un.T @ Un - np.eye(Un.shape[1]))) <= 1e-5


CASES = [(6, 4), (40, 1), (40, 4), (40, 16), (128, 10), (512, 10), (512, 16)]


@pytest.mark.parametrize("wrap", [False, True])
@pytest.mark.parametrize("C", [1, 7, 4096])
@pytest.mark.parametrize("D,k", CASES)
def test_estimator_teacher_forced(D, k, C, wrap):
    steps = max(-(-4 * D // C), 6) + (3 if wrap else 0)
    retained_from = 3 if wrap else 0
    x, g = planted(D, k, steps * C, seed=D + k + C)
    xs, gs = x.reshape(steps, C, D), g.reshape(steps, C, D)
    eng = _engine.get_engine(tf(xs[0]), T.StdNormal(D))
    lw = window(eng, k, xs, gs, retained_from)
    X = xs[retained_from:].reshape(-1, D).astype(np.float64)
    G = gs[retained_from:].reshape(-1, D).astype(np.float64)
    ref = o.compute_low_rank_metric(X, G, C * steps, k, 1e-5, 2.0)
    compare_metric(lw, ref, k)


@pytest.mark.parametrize("growing", [False, True])
def test_update_loop_teacher_forced(growing):
    n, C, D, k = 120, 7, 20, 4
    sched = bj.build_growing_window_schedule(n) if growing else bj.build_schedule(n)
    b = lra.schedule_bytes(sched, n)
    rs = np.random.default_rng(11)
    x, g = planted(D, k, n * C, seed=3)
    xs, gs = x.reshape(n, C, D), g.reshape(n, C, D)
    acc = rs.uniform(0.3, 1.0, (n, C)).astype(F)
    run = o.run_pooled(xs.astype(np.float64), gs.astype(np.float64), acc, sched, max_rank=k, num_steps=n)
    eng = _engine.get_engine(tf(xs[0]), T.StdNormal(D))
    lw = lra._LowRankWindow(eng, k)
    lw.install(1.0)
    hist = torch.empty(n, device=DEV)
    ends = {m[0]: m for m in run.metrics}
    for t in range(n):
        lw.update(tf(xs[t]), tf(gs[t]), tf(acc[t]), b[t], 0.8, 1e-5, 2.0, hist)
        if t in ends:
            compare_metric(lw, ends[t][1:], k)
    np.testing.assert_allclose(npy(hist), run.step_sizes, rtol=1e-5)
    step, mu, _ = lw.final()
    np.testing.assert_allclose(float(step.item()), run.final_step_size, rtol=1e-5)


# ---- the whole warm-up ------------------------------------------------------------------------------------------------
def _run(alg, tgt, x0, key=0, steps=300, **kw):
    warm = bj.window_adaptation_low_rank(alg, tgt, **kw)
    return warm.run(bj.random.key(key, DEV), tf(x0), num_steps=steps)


@pytest.mark.parametrize("alg,extra", [("nuts", {}), ("hmc", {"num_integration_steps": 8})])
def test_runs_on_standard_normal_and_mu_star_recovers_the_mean(alg, extra):
    D, C = 8, 256
    mean = np.linspace(-1.0, 1.0, D)
    tgt = T.DiagGaussian(1.0, dim=D, mean=mean)
    x0 = np.random.default_rng(0).standard_normal((C, D)).astype(F)
    (state, params), info = _run(getattr(bj, alg), tgt, x0, steps=300, max_rank=3, **extra)
    assert 0.0 < params["step_size"] < 10.0
    m = params["inverse_mass_matrix"]
    assert isinstance(m, LowRankMetric) and m.U.shape == (D, 3) and torch.all(m.sigma > 0)
    assert torch.isfinite(info.step_size).all()
    np.testing.assert_allclose(npy(info.mu_star), mean, atol=0.1)
    np.testing.assert_allclose(npy(state.position), np.broadcast_to(npy(info.mu_star), (C, D)), rtol=0, atol=0)
    for key, v in extra.items():
        assert params[key] == v


@pytest.mark.parametrize("rank", [1, 4, 16])
def test_various_ranks(rank):
    D, C = 24, 128
    tgt = T.StdNormal(D)
    x0 = np.random.default_rng(1).standard_normal((C, D)).astype(F)
    (_, params), info = _run(bj.nuts, tgt, x0, steps=200, max_rank=rank)
    m = params["inverse_mass_matrix"]
    assert m.U.shape == (D, rank) and m.lam.shape == (rank,)
    assert np.all(np.isfinite(npy(m.U))) and params["step_size"] > 0


def test_rotated_gaussian_recovered_and_nuts_reproduces_its_moments():
    D, r, C = 256, 10, 1024
    tgt, V, cov = rotated_gaussian(D, r)
    projs, tops = [], []
    for seed in (0, 1):
        x0 = np.random.default_rng(seed).standard_normal((C, D)).astype(F)
        (state, params), info = _run(bj.nuts, tgt, x0, key=seed, steps=400, max_rank=r)
        m = params["inverse_mass_matrix"]
        U, lam = npy(m.U), npy(m.lam)
        # the slow directions (lam < 1 / cutoff) are planted ones; bulk directions may come out just above the cutoff,
        # from the diagonal scaling, as they do in the reference's estimator
        slow = np.argsort(lam)[:int((lam < 0.5).sum())]
        assert len(slow) >= 3, lam
        Us = U[:, slow]
        out = Us - V @ (V.T @ Us)
        assert np.linalg.norm(out) <= 0.2 * np.sqrt(len(slow)), (np.linalg.norm(out), lam)
        projs.append(Us)
        tops.append(U[:, np.argmin(lam)])
    # stable across seeds: the same slow subspace and the same top (slowest) direction, the planted one
    m3 = min(p.shape[1] for p in projs)
    P0, P1 = (p[:, :m3] @ p[:, :m3].T for p in projs)
    assert np.linalg.norm(P0 - P1) < 0.5, np.linalg.norm(P0 - P1)
    assert abs(tops[0] @ tops[1]) > 0.95
    assert abs(tops[0] @ V[:, 0]) > 0.95
    # NUTS with the adapted parameters, after 100 steps away from the common start mu*: mean and variance within 5 MCSE
    state, _, _, _ = bj.sample_nuts_native(bj.random.key(8, DEV), state, tgt, params["step_size"], m, 100,
                                           keep_history=False)
    _, hist, _, _ = bj.sample_nuts_native(bj.random.key(9, DEV), state, tgt, params["step_size"], m, 200)
    ess = npy(bj.diagnostics.effective_sample_size(hist, tgt))
    h = npy(hist)
    mean = h.mean((0, 1))
    var = h.var((0, 1))
    sd = np.sqrt(np.diag(cov))
    assert np.all(np.abs(mean) <= 5 * sd / np.sqrt(ess)), np.max(np.abs(mean) / (sd / np.sqrt(ess)))
    # the variance's MCSE from the ESS of the squared draws (the target's mean is zero)
    ess2 = npy(bj.diagnostics.effective_sample_size((hist * hist).contiguous(), tgt))
    assert np.all(np.abs(var - np.diag(cov)) <= 5 * np.sqrt(2.0) * np.diag(cov) / np.sqrt(ess2))


def test_two_runs_are_bit_identical():
    D, C = 40, 512
    tgt = T.StdNormal(D)
    x0 = np.random.default_rng(2).standard_normal((C, D)).astype(F)
    (s1, p1), i1 = _run(bj.nuts, tgt, x0, key=4, steps=200, max_rank=4)
    (s2, p2), i2 = _run(bj.nuts, tgt, x0, key=4, steps=200, max_rank=4)
    assert p1["step_size"] == p2["step_size"]
    for a, b in zip(p1["inverse_mass_matrix"], p2["inverse_mass_matrix"]):
        assert torch.equal(a, b)
    assert torch.equal(i1.state.position, i2.state.position)
    assert torch.equal(i1.step_size, i2.step_size) and torch.equal(i1.mu_star, i2.mu_star)


def test_rejections():
    x0 = np.zeros((8, 600), F)
    with pytest.raises(ValueError):
        _run(bj.nuts, T.StdNormal(600), x0, steps=30)
    # transitions off the warp kernels: the dense path
    with pytest.raises(BjxError):
        _run(bj.nuts, T.DenseGaussian(np.eye(256) * 2.0), np.zeros((8, 256), F), steps=30)
    with pytest.raises(NotImplementedError):
        bj.window_adaptation_low_rank(bj.nuts, T.StdNormal(4), buffer_policy="accumulating")
    with pytest.raises(NotImplementedError):
        bj.window_adaptation_low_rank(bj.nuts, T.StdNormal(4), gradient_based_init=True)
    with pytest.raises(ValueError):
        bj.window_adaptation_low_rank(bj.nuts, T.StdNormal(4), max_rank=17)
