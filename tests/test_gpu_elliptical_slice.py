"""Elliptical slice sampling on the GPU: one teacher-forced transition against the float32 oracle
(oracle/elliptical_slice.py) in every row size class, on the tensor-core route and on the CTA rows; the cap path; the
native loops bit-identical to step calls on all three routes; chain_offset and plug-in bit identity; the rejections; and
posterior moments within 5 MCSE.

theta, subiter and exhausted must match the oracle exactly except on chains where one of the oracle's loop decisions
was a tie: |logL(p) - logy| below TIE_REL * (1 + |logy| + D), twice that with a dense prior.  The device's cos / sin
and the oracle's NumPy ones may differ in the last bit, and the dense prior's L z is summed in another order (or by the
float32-accurate tensor-core product): either moves logL(p) by about 1e-7 to 1e-6 of the size of its terms."""
import numpy as np
import pytest
import torch

import blackjax_b200 as bj
from blackjax_b200 import _lib
from oracle import elliptical_slice as oe
from oracle import prng as oprng
from oracle import targets as otargets
from test_gpu_parity import close, make_target, npy, tf, tk

pytestmark = pytest.mark.gpu
F = np.float32
TIE_REL = 3e-6


def spd(D, rs, scale=1.0):
    A = rs.standard_normal((D, D))
    return (scale * (A @ A.T / D + 0.5 * np.eye(D))).astype(F)


def make_prior(prior, mean_kind, D, rs):
    mean = F(0.2) if mean_kind == "scalar" else (0.3 * rs.standard_normal(D)).astype(F)
    cov = np.exp(rs.uniform(-0.5, 0.5, D)).astype(F) if prior == "diag" else spd(D, rs)
    return mean, cov


def run_step(tgt, q, keys, mean, cov, max_subiter=1000):
    """One transition through Engine.elliptical_slice_step with every info field; returns the device's (q, logl, info)
    and the start log-likelihood (the oracle starts from the same state)."""
    from blackjax_b200._engine import get_engine
    st = bj.elliptical_slice.init(tf(q), tgt)
    eng = get_engine(st.position, tgt)
    eng.ensure_elliptical_prior(tf(np.asarray(mean, F)), tf(cov))
    C, D = q.shape
    f = dict(momentum=torch.empty(C, D, device="cuda"), theta=torch.empty(C, device="cuda"),
             subiter=torch.empty(C, dtype=torch.int32, device="cuda"),
             exhausted=torch.empty(C, dtype=torch.uint8, device="cuda"))
    qo, lo = eng.elliptical_slice_step(tk(keys), *st, max_subiter, info_fields=f)
    torch.cuda.synchronize()
    return npy(qo), npy(lo), {k: npy(v) for k, v in f.items()}, npy(st.logdensity)


def compare(keys, q, l0, otgt, mean, cov, got, max_subiter=1000, row_max=False):
    qd, ld, info, _ = got
    C, D = q.shape
    (qo, lo), oinfo = oe.step(keys, q, l0, otgt, mean, oe.prior_scale(cov), max_subiter)
    with np.errstate(divide="ignore", invalid="ignore"):
        logy = np.abs(l0.astype(np.float64) + np.log(oprng.uniform(oprng.split(keys, 4)[:, 2]).astype(np.float64)))
    tie = TIE_REL * (2.0 if row_max else 1.0) * (1.0 + np.where(np.isfinite(logy), logy, 0.0) + D)
    ok = oinfo["margin"] > tie
    assert ok.mean() >= 0.8, f"{(~ok).sum()} of {C} chains tie"
    np.testing.assert_array_equal(info["subiter"][ok], oinfo["subiter"][ok])
    np.testing.assert_array_equal(info["exhausted"][ok].astype(bool), oinfo["exhausted"][ok])
    np.testing.assert_array_equal(info["theta"][ok], oinfo["theta"][ok])
    ff = 1.0 if row_max else None
    for a, b in ((qd, qo), (info["momentum"], oinfo["momentum"])):
        for c in np.nonzero(ok)[0]:
            close(a[c], b[c], floor_frac=ff)
    close(ld[ok], lo[ok], scale=np.abs(lo[ok]).max() + D)
    return oinfo, ok


# (target, D, prior, mean): every row size class (1, 2, 3: S1; 31: S1; 100: S4; 128: V1; 256: V2; 1024: V8), the
# dense prior in the warp (<= 128) and on the tensor-core route (256, 1024), scalar and [D] means
CASES = [("std", 1, "diag", "scalar"), ("banana", 2, "diag", "vec"), ("banana", 2, "dense", "scalar"),
         ("funnel", 3, "dense", "vec"), ("diag", 31, "dense", "vec"), ("funnel", 100, "diag", "scalar"),
         ("dense", 100, "dense", "vec"), ("dense", 128, "diag", "vec"), ("diag", 128, "dense", "scalar"),
         ("funnel", 256, "diag", "vec"), ("diag", 256, "dense", "vec"), ("funnel", 512, "diag", "scalar"),
         ("diag", 1024, "diag", "scalar"), ("funnel", 1024, "dense", "vec"), ("std", 1024, "dense", "scalar"),
         # CTA rows: the smallest big row, a middle one and the largest (18432 dims)
         ("diag", 1028, "diag", "vec"), ("funnel", 2048, "diag", "scalar"), ("std", 18432, "diag", "vec")]


def start(kind, D, rs):
    q = (0.5 * rs.standard_normal((1, D))).astype(F)
    if kind == "funnel":
        q[:, 0] = 0.0
    return q


@pytest.mark.parametrize("kind, D, prior, mean_kind", CASES)
def test_single_transition_matches_oracle(kind, D, prior, mean_kind):
    rs = np.random.default_rng(D + len(kind))
    C = 256 if D <= 1024 else 32
    tgt, otgt = make_target(kind, D, rs)
    mean, cov = make_prior(prior, mean_kind, D, rs)
    q = np.concatenate([start(kind, D, rs) for _ in range(C)])
    keys = oprng.split(oprng.key(D), C)
    got = run_step(tgt, q, keys, mean, cov)
    compare(keys, q, got[3], otgt, mean, cov, got, row_max=prior == "dense")


def test_hier_logit_10000_matches_oracle():
    """BASELINE config 5's hierarchical logistic regression on the CTA rows, teacher-forced."""
    C, D = 6, 10000
    x, bits = bj.targets.HierLogit.synthetic_data(D - 4, seed=1)
    tgt, otgt = bj.targets.HierLogit(x, bits), otargets.HierLogit(x, bits)
    rs = np.random.default_rng(3)
    q = (0.3 * rs.standard_normal((C, D))).astype(F)
    mean, cov = F(0.0), np.full(D, 0.25, F)
    keys = oprng.split(oprng.key(4), C)
    got = run_step(tgt, q, keys, mean, cov)
    compare(keys, q, got[3], otgt, mean, cov, got)


@pytest.mark.parametrize("max_subiter", [1, 2])
@pytest.mark.parametrize("D, prior", [(64, "diag"), (64, "dense"), (256, "dense"), (2048, "diag")])
def test_cap_path_matches_oracle(max_subiter, D, prior):
    """A likelihood much narrower than the prior: many first proposals fall below the slice, so with max_subiter = 1 or
    2 many chains end exhausted, keep their state and report theta = 0 and momentum = nu (compare() holds the momentum
    to the oracle's, which is nu there)."""
    rs = np.random.default_rng(7)
    C = 256 if D <= 1024 else 16
    tgt = bj.targets.DiagGaussian(np.full(D, 0.3), mean=np.zeros(D, F))
    otgt = otargets.DiagGaussian(np.full(D, 0.3), mean=np.zeros(D, F))
    mean, cov = make_prior(prior, "vec", D, rs)
    q = (0.3 * rs.standard_normal((C, D))).astype(F)
    keys = oprng.split(oprng.key(9), C)
    got = run_step(tgt, q, keys, mean, cov, max_subiter)
    oinfo, ok = compare(keys, q, got[3], otgt, mean, cov, got, max_subiter, row_max=prior == "dense")
    ex = got[2]["exhausted"].astype(bool) & ok
    assert ex.sum() >= 4
    np.testing.assert_array_equal(got[0][ex], q[ex])
    assert np.all(got[2]["theta"][ex] == 0) and np.all(got[2]["subiter"][ex] == max_subiter)


def stepwise(key, st, tgt, mean, cov, T_, thin, chain_offset, max_subiter=1000):
    kern = bj.elliptical_slice.build_kernel(cov, mean, max_subiter, chain_offset=chain_offset)
    hist, sub = [], []
    for t, k in enumerate(oprng.split(key, T_)):
        st, info = kern(tk(k), st, tgt)
        sub.append(npy(info.subiter))
        if (t + 1) % thin == 0:
            hist.append(npy(st.position))
    return st, np.stack(hist), np.stack(sub)


@pytest.mark.parametrize("D, prior", [(100, "diag"), (64, "dense"), (256, "dense"), (2048, "diag")])
def test_native_loop_bit_identical_to_steps(D, prior):
    """All three routes: the warp rows (diagonal and small dense prior), the tensor-core route and the CTA rows."""
    rs = np.random.default_rng(5)
    C, T_, thin, off = 40, 10, 3, 7
    tgt, _ = make_target("diag", D, rs)
    mean, cov = make_prior(prior, "vec", D, rs)
    mean, cov = tf(mean), tf(cov)
    q = tf((0.5 * rs.standard_normal((C, D))).astype(F))
    key = oprng.key(21)
    st0 = bj.elliptical_slice.init(q, tgt)
    ref, h_ref, s_ref = stepwise(key, st0, tgt, mean, cov, T_, thin, off)
    fin, hist, sub = bj.sample_elliptical_slice_native(tk(key), st0, tgt, mean, cov, T_, thin=thin, chain_offset=off)
    np.testing.assert_array_equal(npy(fin.position), npy(ref.position))
    np.testing.assert_array_equal(npy(fin.logdensity), npy(ref.logdensity))
    np.testing.assert_array_equal(npy(hist), h_ref)
    np.testing.assert_array_equal(npy(sub), s_ref)
    assert s_ref.max() > 1


def test_chain_offset_split_matches_one_handle():
    """One shared key over 64 chains on one handle equals two handles of 32 chains with chain_offset 0 and 32."""
    rs = np.random.default_rng(8)
    D, C = 96, 64
    tgt, _ = make_target("diag", D, rs)
    mean, cov = (tf(a) for a in make_prior("diag", "vec", D, rs))
    q = tf((0.5 * rs.standard_normal((C, D))).astype(F))
    key = tk(oprng.key(3))
    whole = bj.sample_elliptical_slice_native(key, bj.elliptical_slice.init(q, tgt), tgt, mean, cov, 6)
    for lo in (0, 32):
        part = bj.sample_elliptical_slice_native(key, bj.elliptical_slice.init(q[lo:lo + 32].clone(), tgt), tgt, mean,
                                                 cov, 6, chain_offset=lo)
        assert torch.equal(part[0].position, whole[0].position[lo:lo + 32])
        assert torch.equal(part[1], whole[1][:, lo:lo + 32])
        assert torch.equal(part[2], whole[2][:, lo:lo + 32])


def test_plugins_match_builtin():
    """The diag_gaussian plug-in against StdNormal (rows) and diag_gaussian_big against it at D = 2048 (CTA rows):
    bit-identical native loops."""
    from blackjax_b200 import plugin
    for D, src in ((100, "diag_gaussian"), (2048, "diag_gaussian_big")):
        C = 32
        user = bj.targets.UserTarget(D, plugin.read_example(src), np.ones(D, F), name=src)
        builtin = bj.targets.StdNormal(D)
        q = tf(np.random.default_rng(D).standard_normal((C, D)).astype(F))
        mean, cov = tf(np.zeros(D, F)), tf(np.full(D, 2.0, F))
        key = tk(oprng.key(5))
        a = bj.sample_elliptical_slice_native(key, bj.elliptical_slice.init(q.clone(), builtin), builtin, mean, cov, 6)
        b = bj.sample_elliptical_slice_native(key, bj.elliptical_slice.init(q.clone(), user), user, mean, cov, 6)
        assert torch.equal(a[0].position, b[0].position) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])


def test_rejections():
    from blackjax_b200._engine import get_engine
    C = 4
    k = tk(oprng.split(oprng.key(0), C))
    # a call before bjx_set_elliptical_prior
    tgt = bj.targets.StdNormal(8)
    st = bj.elliptical_slice.init(tf(np.zeros((C, 8), F)), tgt)
    with pytest.raises(_lib.BjxError, match="needs a prior"):
        get_engine(st.position, tgt).elliptical_slice_step(k, *st, 10)
    # a dense prior beyond 1024 dims (rows beyond 128 dims with dim % 4 != 0 have no size class at all)
    D = 1028
    tgt = bj.targets.StdNormal(D)
    st = bj.elliptical_slice.init(tf(np.zeros((C, D), F)), tgt)
    with pytest.raises(_lib.BjxError, match="dim <= 1024"):
        bj.elliptical_slice.build_kernel(tf(np.eye(D, dtype=F)), 0.0)(k, st, tgt)
    # a dense Gaussian target beyond 128 dims (the tensor-core target path)
    D = 256
    tgt = bj.targets.DenseGaussian(spd(D, np.random.default_rng(1)))
    st = bj.elliptical_slice.init(tf(np.zeros((C, D), F)), tgt)
    with pytest.raises(_lib.BjxError, match="tensor-core dense target path"):
        bj.elliptical_slice.build_kernel(tf(np.ones(D, F)), 0.0)(k, st, tgt)
    # a dense prior that is not positive definite
    tgt = bj.targets.StdNormal(8)
    st = bj.elliptical_slice.init(tf(np.zeros((C, 8), F)), tgt)
    with pytest.raises(_lib.BjxError, match="not positive definite"):
        bj.elliptical_slice.build_kernel(tf(-np.eye(8, dtype=F)), 0.0)(k, st, tgt)


def mcse_check(h, mean, var, tgt):
    """Posterior mean and variance of every dimension within 5 MCSE, with the device ESS of the draws (and of their
    squared deviations for the variance)."""
    from blackjax_b200.diagnostics import effective_sample_size
    x = h.double()
    mean, var = np.array(mean), np.array(var)
    d2 = ((x - torch.as_tensor(mean, device=x.device).double()) ** 2)
    ess = effective_sample_size(h, tgt).double()
    ess2 = effective_sample_size(d2.float().contiguous(), tgt).double()
    m = x.mean(dim=(0, 1))
    v = d2.mean(dim=(0, 1))
    sd = x.std(dim=(0, 1))
    sd2 = d2.std(dim=(0, 1))
    zm = ((m - torch.as_tensor(mean, device=x.device).double()).abs() / (sd / ess.sqrt())).cpu().numpy()
    zv = ((v - torch.as_tensor(var, device=x.device).double()).abs() / (sd2 / ess2.sqrt())).cpu().numpy()
    assert zm.max() < 5, zm.max()
    assert zv.max() < 5, zv.max()


def test_flat_likelihood_recovers_prior():
    """test_sampling.py:1148-1157: a flat likelihood (a zero-precision diagonal Gaussian) with the prior N(1, 4)."""
    C, T_ = 4096, 300
    tgt = bj.targets.DiagGaussian(np.array([1e30]))  # inv_var rounds to 0 in float32: logL = 0
    st = bj.elliptical_slice.init(tf(np.zeros((C, 1), F)), tgt)
    _, hist, sub = bj.sample_elliptical_slice_native(tk(oprng.key(1)), st, tgt, 1.0, tf(np.array([4.0], F)), T_)
    assert int(sub.max()) == 1  # the first proposal is always above the slice of a flat likelihood
    mcse_check(hist[50:].contiguous(), np.array([1.0]), np.array([4.0]), tgt)


@pytest.mark.parametrize("D", [64, 256])
def test_conjugate_gaussian_posterior(D):
    """Dense prior N(m0, S0) times the diagonal Gaussian likelihood N(mu_l, diag(s^2)): the posterior is Gaussian with
    covariance S = (S0^-1 + diag(s^-2))^-1 and mean S (S0^-1 m0 + diag(s^-2) mu_l).  D = 256 takes the tensor-core
    route."""
    rs = np.random.default_rng(D)
    C, T_ = 2048, 200
    s = np.exp(rs.uniform(-0.3, 0.3, D))
    mu_l = rs.standard_normal(D)
    S0 = spd(D, rs).astype(np.float64)
    m0 = 0.5 * rs.standard_normal(D)
    tgt = bj.targets.DiagGaussian(s, mean=mu_l.astype(F))
    P = np.linalg.inv(S0.astype(F).astype(np.float64)) + np.diag(1.0 / (s.astype(F).astype(np.float64) ** 2))
    S = np.linalg.inv(P)
    mpost = S @ (np.linalg.solve(S0.astype(F).astype(np.float64), m0.astype(F)) + mu_l.astype(F) / s.astype(F) ** 2)
    # the chains start at exact posterior draws, so that every draw is from the stationary distribution: elliptical slice
    # sampling mixes slowly here (an ESS of about 1 % of the draws at D = 64), and a burn-in would have to be long
    x0 = mpost + rs.standard_normal((C, D)) @ np.linalg.cholesky(S).T
    st = bj.elliptical_slice.init(tf(x0.astype(F)), tgt)
    _, hist, _ = bj.sample_elliptical_slice_native(tk(oprng.key(2)), st, tgt, tf(m0.astype(F)), tf(S0.astype(F)), T_)
    mcse_check(hist, mpost, np.diag(S), tgt)
