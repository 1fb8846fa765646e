"""Random-walk Metropolis: the float32 oracle (oracle/random_walk.py) against the reference's known answers
(tests/mcmc/test_random_walk_without_chex.py), explicit compositions of the key tree and the energies, the Python API
surface and its descriptors, and the ptxas report of the new kernels.  No GPU needed."""
import inspect
import os
import re

import numpy as np
import pytest

from oracle import prng
from oracle import random_walk as orw
from oracle.targets import StdNormal
from test_kernel_spills import CLEAN, INSTANCES, NVCC, ptxas_log

F = np.float32


def test_one_step_addition():
    """test_one_step_addition: a step of +10 from 50 to a log-density that is higher past 59 is accepted to 60; the
    stored log-density 1.0 is used as given."""
    def logdensity(x):
        return np.where(np.all(x > 59.0, axis=1), F(0.0), F(0.5)).astype(F), None

    (x, lp), info = orw.step(prng.key(0)[None], np.array([[50.0]], F), F(1.0), logdensity,
                             proposal=lambda k, x: (x + F(10.0)).astype(F))
    np.testing.assert_allclose(x, [[60.0]])
    assert info["is_accepted"][0] and lp[0] == 0.0


def irmh_logdensity(x):
    return np.where(np.all(x - 10.0 < 1e-10, axis=1), F(0.0), F(0.5)).astype(F), None


@pytest.mark.parametrize("x0", [50.0, 15000.0])
def test_irmh_is_independent_of_position(x0):
    """test_proposal_is_independent_of_position: the candidate is 10 from any position, accepted with rate e^-1."""
    (x, _), info = orw.step(prng.key(0)[None], np.array([[x0]], F), F(1.0), irmh_logdensity,
                            proposal=lambda k, x: np.full_like(x, 10.0))
    np.testing.assert_allclose(x, [[10.0]])
    np.testing.assert_allclose(info["acceptance_rate"], 0.367879, rtol=1e-5)


def test_irmh_non_symmetric_proposal():
    """test_non_symmetric_proposal: proposal_logdensity_fn enters both energies, acceptance exp(-1.4)."""
    def f(new, prev):
        return np.where(np.all(new[0] - 10 < 1e-10, axis=1), F(0.1), F(0.5)).astype(F)

    _, info = orw.step(prng.key(0)[None], np.array([[50.0]], F), F(1.0), irmh_logdensity,
                       proposal=lambda k, x: np.full_like(x, 10.0), proposal_logdensity_fn=f)
    np.testing.assert_allclose(info["acceptance_rate"], 0.246597, rtol=1e-6)


def test_transition_energy():
    """test_energy: E(a, b) = -logp(b) without a correction, -logp(b) - f(b, a) with one."""
    one, another = (np.zeros((1, 1), F), F(50.0)), (np.ones((1, 1), F), F(30.0))

    def f(new, prev):
        return F(100.0) if new is one else F(200.0)

    def energy(prev, new, fn):
        return -new[1] - (fn(new, prev) if fn else F(0.0))

    assert energy(one, another, None) == -30.0 and energy(another, one, None) == -50.0
    assert energy(one, another, f) == -230.0 and energy(another, one, f) == -150.0


@pytest.mark.parametrize("sigma", [F(0.7), np.array([0.5, 2.0, 1.0], F),
                                   np.array([[1.0, 0.0, 0.0], [0.5, 2.0, 0.0], [0.1, 0.2, 0.5]], F)])
@pytest.mark.parametrize("mean", [None, np.array([1.0, -1.0, 0.5], F)])
def test_key_tree_composed_explicitly(sigma, mean):
    """The candidate from normal(split(key)[0]) and the decision from uniform(split(key)[1]), composed from oracle.prng
    and linear_map."""
    C, D = 5, 3
    keys = prng.split(prng.key(4), C)
    x = np.random.default_rng(0).standard_normal((C, D)).astype(F)
    fn = StdNormal(D)
    lp = fn(x)[0]
    (xn, ln), info = orw.step(keys, x, lp, fn, sigma=sigma, mean=mean)
    z = np.stack([prng.normal(prng.fold_in(k, 0), (D,)) for k in keys])
    lin = (sigma * z) if np.ndim(sigma) <= 1 else (z.astype(np.float64) @ sigma.T.astype(np.float64))
    y = ((x if mean is None else mean) + lin.astype(F)).astype(F)
    np.testing.assert_array_equal(info["candidate"][0], y)
    la = (fn(y)[0] - lp).astype(F)
    np.testing.assert_array_equal(info["log_a"], la)
    u = np.array([prng.uniform(prng.fold_in(k, 1)) for k in keys])
    np.testing.assert_array_equal(info["is_accepted"], u < np.minimum(np.exp(la), 1))
    np.testing.assert_array_equal(xn, np.where(info["is_accepted"][:, None], y, x))


def test_gaussian_correction_is_the_log_ratio_of_proposal_densities():
    """gaussian_logdensity(mean, sigma) in the energies: log_a = logp(y) - logp(x) + log q(x) - log q(y) for the
    independent proposal q = N(mean, diag(sigma)^2), to float32 rounding."""
    from scipy import stats
    C, D = 64, 4
    mean, sigma = np.array([0.5, -1.0, 0.0, 2.0], F), np.array([1.5, 0.7, 2.0, 1.0], F)
    x = np.random.default_rng(1).standard_normal((C, D)).astype(F)
    fn = StdNormal(D)
    _, info = orw.step(prng.split(prng.key(5), C), x, fn(x)[0], fn, sigma=sigma, mean=mean,
                       proposal_logdensity_fn=orw.gaussian_logdensity(mean, sigma))
    y = info["candidate"][0].astype(np.float64)
    q = stats.norm(mean.astype(np.float64), sigma.astype(np.float64))
    want = (fn(y.astype(F))[0].astype(np.float64) - fn(x)[0] + q.logpdf(x).sum(1) - q.logpdf(y).sum(1))
    np.testing.assert_allclose(info["log_a"], want, rtol=1e-5, atol=1e-4)


def test_correction_removes_the_independent_proposal_bias():
    """N(0, 1) with the independent proposal N(0, 2^2): with the correction the chains target N(0, 1); without it the
    stationary law is N(0, 0.8), the target times the proposal density."""
    C, T = 4000, 60
    fn = StdNormal(1)
    for corr, var in ((orw.gaussian_logdensity(0.0, 2.0), 1.0), (None, 0.8)):
        x = np.zeros((C, 1), F)
        lp = fn(x)[0]
        draws = []
        for k in prng.split(prng.key(11), T):
            (x, lp), _ = orw.step(prng.split(k, C), x, lp, fn, sigma=F(2.0), mean=F(0.0), proposal_logdensity_fn=corr)
            draws.append(x[:, 0].copy())
        v = np.var(np.array(draws[20:]))
        assert abs(v - var) < 0.05, (corr is not None, v)


def test_nan_candidate_is_rejected():
    def fn(q):
        return np.where(np.abs(q[:, 0]) < 0.1, F(0.0), F(np.nan)).astype(F), None

    x = np.zeros((16, 1), F)
    (xn, ln), info = orw.step(prng.split(prng.key(2), 16), x, np.zeros(16, F), fn, sigma=F(5.0))
    nan = np.isnan(info["candidate"][1])
    assert nan.any() and not info["is_accepted"][nan].any() and (info["acceptance_rate"][nan] == 0).all()
    np.testing.assert_array_equal(xn[nan], x[nan])


def test_api_surface():
    import blackjax_b200 as bj
    from blackjax_b200.mcmc import random_walk as rw
    assert callable(bj.sample_random_walk_native)
    assert bj.additive_step_random_walk.normal_random_walk is rw.normal_random_walk
    assert bj.rmh.build_kernel is rw.build_rmh and bj.irmh.build_kernel is rw.build_irmh
    assert bj.additive_step_random_walk.build_kernel is rw.build_additive_step and bj.rmh.init is rw.init
    assert rw.RWState._fields == ("position", "logdensity")
    assert rw.RWInfo._fields == ("acceptance_rate", "is_accepted", "proposal")
    assert list(inspect.signature(rw.rmh_as_top_level_api).parameters) == ["logdensity_fn", "proposal_generator",
                                                                          "proposal_logdensity_fn"]
    assert list(inspect.signature(rw.irmh_as_top_level_api).parameters) == ["logdensity_fn", "proposal_distribution",
                                                                           "proposal_logdensity_fn"]
    assert list(inspect.signature(rw.build_rmh).parameters) == ["inplace", "chain_offset"]
    with pytest.raises(ValueError, match="vector or a matrix"):
        rw.normal(np.zeros((2, 2, 2)))
    with pytest.raises(NotImplementedError, match="gaussian_proposal"):
        bj.rmh(lambda x: x, lambda k, p: p)
    with pytest.raises(NotImplementedError, match="gaussian_distribution"):
        bj.irmh(lambda x: x, lambda k: 0.0)
    with pytest.raises(ValueError, match="must be normal"):
        bj.additive_step_random_walk(lambda x: x, rw.gaussian_proposal(1.0))
    with pytest.raises(ValueError, match="must be gaussian_proposal"):
        bj.rmh(lambda x: x, rw.normal(1.0))
    # the correction pairs only with a position-independent proposal of the same mean and sigma
    bj.irmh(lambda x: x, rw.gaussian_distribution(1.0, 2.0), rw.gaussian_logdensity(1.0, 2.0))
    bj.rmh(lambda x: x, rw.gaussian_proposal(2.0, mean=1.0), rw.gaussian_logdensity(1.0, 2.0))
    for bad in (lambda: bj.irmh(lambda x: x, rw.gaussian_distribution(1.0, 2.0), rw.gaussian_logdensity(0.0, 2.0)),
                lambda: bj.rmh(lambda x: x, rw.gaussian_proposal(2.0), rw.gaussian_logdensity(0.0, 2.0))):
        with pytest.raises(ValueError, match="corrects only"):
            bad()
    with pytest.raises(NotImplementedError, match="proposal_logdensity_fn"):
        bj.irmh(lambda x: x, rw.gaussian_distribution(1.0, 2.0), lambda new, prev: 0.0)
    with pytest.raises(ValueError, match="dense sigma"):
        rw.gaussian_logdensity(0.0, np.eye(2))


# the instances of test_kernel_spills.py with the velocity Verlet form, the small dense sigma's (dm) instances where
# the library builds them (dim <= 128), and the CTA-row kernel of every built-in big-row target
SMALL = ("Row<1, false>", "Row<4, false>", "Row<4, true>")
ROW_INSTANCES = [(r, tk, "false") for r, tk in INSTANCES] + [(r, tk, "true") for r, tk in INSTANCES if r in SMALL]
BIG_TARGETS = ["BJX_TARGET_DIAG_GAUSSIAN", "BJX_TARGET_FUNNEL", "BJX_TARGET_HIER_LOGIT"]


@pytest.mark.skipif(not os.path.exists(NVCC), reason="needs nvcc")
def test_kernels_compile_without_spills(tmp_path):
    """k_rw_transition, k_rw_chains and k_big_rw compile with no stack frame and no spills (ptxas -v)."""
    lines = ['#include "bjx_big.cuh"', "namespace bjx {"]
    for row, tk, dm in ROW_INSTANCES:
        lines.append(f"template __global__ void k_rw_transition<{row}, {tk}, {dm}>(Params, const uint32_t*, "
                     "const float*, const float*, float*, float*, RwArgs);")
        lines.append(f"template __global__ void k_rw_chains<{row}, {tk}, {dm}>(Params, float*, float*, RwArgs);")
    for tk in BIG_TARGETS:
        lines.append(f"template __global__ void k_big_rw<{tk}>(BigParams, const uint32_t*, const float*, const float*, "
                     "float*, float*, RwArgs);")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    log = ptxas_log(tmp_path, "\n".join(lines + ["}"]) + "\n",
                    ["-Xptxas", "-v", "-I", os.path.join(root, "blackjax_b200", "csrc"), "-I",
                     os.path.join(root, "include")])
    blocks = [b for b in re.split(r"Compiling entry function", log) if "_rw" in b.split("\n")[0]]
    assert len(blocks) == 2 * len(ROW_INSTANCES) + len(BIG_TARGETS), [b.split("\n")[0] for b in blocks]
    bad = [" ".join(b.split("\n")[:3]) for b in blocks if CLEAN not in b]
    assert not bad, "\n".join(bad)
