"""Random-walk Metropolis on the GPU: one transition of the additive step, rmh (position-relative and
position-independent) and irmh against the float32 oracle (oracle/random_walk.py) in every row size class and on the CTA
rows, with and without the proposal correction; rejected and NaN candidates; the plug-ins; the native loops
bit-identical to step calls; the reference's univariate-normal statistics; the correction's effect; and the refusals.

Decision rule (as test_gpu_big_rows.compare_transition): the device's log-densities and correction sums round
differently from the oracle's, by up to DE_REL of the size of their terms.  Acceptance rates must agree within that
error, and decisions must be equal except where the oracle's log u lies within twice that error of min(log_a, 0)."""
import numpy as np
import pytest
import torch

import blackjax_b200 as bj
from blackjax_b200 import _lib
from blackjax_b200.mcmc import random_walk as rw
from oracle import prng as oprng
from oracle import random_walk as orw
from oracle import targets as otargets
from test_gpu_parity import close, make_target, npy, tf, tk

pytestmark = pytest.mark.gpu
F = np.float32
DE_REL = 1e-5


def make_sigma(kind, D, scale, rs):
    if kind == "scalar":
        return F(scale)
    if kind == "vec":
        return (scale * np.exp(rs.uniform(-0.3, 0.3, D))).astype(F)
    A = rs.standard_normal((D, D))
    return (scale * np.linalg.cholesky(A @ A.T / D + 0.5 * np.eye(D))).astype(F)


def descriptors(mode, sigma, mean, correct):
    """(kernel builder, proposal descriptor, correction or None) of a mode."""
    corr = rw.gaussian_logdensity(mean, sigma) if correct else None
    if mode == "additive":
        return rw.build_additive_step, rw.normal(sigma), None
    if mode == "rmh":
        return rw.build_rmh, rw.gaussian_proposal(sigma), None
    if mode == "rmh_ind":
        return rw.build_rmh, rw.gaussian_proposal(sigma, mean=mean), corr
    return rw.build_irmh, rw.gaussian_distribution(mean, sigma), corr


def run_step(tgt, q, keys, mode, sigma, mean, correct, inplace=False):
    st = rw.init(tf(q), tgt)
    before = tuple(t.clone() for t in st)
    build, prop, corr = descriptors(mode, sigma if np.ndim(sigma) == 0 else tf(sigma),
                                    None if mean is None else tf(mean), correct)
    kern = build(inplace=inplace)
    new, info = kern(tk(keys), st, tgt, prop) if corr is None else kern(tk(keys), st, tgt, prop, corr)
    torch.cuda.synchronize()
    if inplace:
        assert new.position.data_ptr() == st.position.data_ptr()
    assert new.position.data_ptr() == info.proposal.position.data_ptr()  # proposal: the post-accept state
    return new, info, before


def compare(keys, q, otgt, mode, sigma, mean, correct, new, info, before):
    """The device transition against the oracle's; returns the device decisions."""
    C, D = q.shape
    lp0 = npy(before[1])
    ind = mode in ("rmh_ind", "irmh")
    (xo, lo), oi = orw.step(keys, q, lp0, otgt, sigma=sigma, mean=mean if ind else None,
                            proposal_logdensity_fn=orw.gaussian_logdensity(mean, sigma) if correct else None)
    y, ly = oi["candidate"]
    terms = np.abs(lp0) + np.where(np.isfinite(ly), np.abs(ly), 0) + D
    if correct:
        inv = F(1.0) / np.asarray(sigma, F)
        terms = terms + 0.5 * (np.sum(((q - mean) * inv) ** 2, 1) + np.sum(((y - mean) * inv) ** 2, 1))
    de = DE_REL * terms
    with np.errstate(invalid="ignore"):
        near = np.abs(oi["log_u"] - np.minimum(oi["log_a"], 0)) <= 2 * de
    pa, acc = npy(info.acceptance_rate), npy(info.is_accepted).astype(bool)
    assert (np.abs(pa - oi["acceptance_rate"]) <= 1e-5 + 2 * de * oi["acceptance_rate"]).all(), \
        np.max(np.abs(pa - oi["acceptance_rate"]))
    assert ((acc == oi["is_accepted"]) | near).all()
    a = acc & oi["is_accepted"]
    dense = np.ndim(sigma) == 2
    close(npy(new.position)[a], y[a], rtol=2e-5 if dense else 1e-5)
    close(npy(new.logdensity)[a], ly[a], scale=np.max(np.abs(ly[a]), initial=0) + D)
    # a rejected chain carries its input over bit for bit, in place or out of place
    r = torch.from_numpy(~acc).to(new.position.device)
    for got, was in zip(new, before):
        assert torch.equal(got[r], was[r])
    return acc, oi


# (target, D, sigma kind, mode, correct, in place): every row size class, every mode and sigma kind, the CTA rows
MODES = ["additive", "rmh", "rmh_ind", "irmh"]
CASES = ([("std", 1, "scalar", m, c, ip) for m, c, ip in (("additive", False, False), ("rmh", False, True),
                                                            ("rmh_ind", True, False), ("irmh", True, True),
                                                            ("irmh", False, False))]
         + [("diag", 64, "dense", m, False, m == "rmh") for m in MODES]
         + [("funnel", 64, "vec", m, m in ("rmh_ind", "irmh"), m == "irmh") for m in MODES]
         + [("dense", 128, "dense", m, False, m == "additive") for m in MODES]
         + [("diag", 128, "vec", "irmh", True, False), ("banana", 2, "scalar", "rmh", False, False),
            ("std", 33, "vec", "rmh_ind", True, True), ("diag", 516, "scalar", "additive", False, False)]
         + [("diag", 1024, k, m, c, False) for k, m, c in (("vec", "additive", False), ("scalar", "irmh", True),
                                                          ("vec", "rmh_ind", False))]
         + [("diag", 2048, "vec", m, m in ("rmh_ind", "irmh"), m == "additive") for m in MODES]
         + [("funnel", 2048, "scalar", "additive", False, True), ("std", 10756, "vec", "irmh", True, False),
            ("std", 10756, "scalar", "rmh", False, True), ("std", 18432, "vec", "additive", False, False),
            ("diag", 18432, "scalar", "rmh_ind", True, True)])


def start(kind, D, C, rs, otgt):
    q = (0.7 * rs.standard_normal((C, D))).astype(F)
    if kind == "funnel":
        q[:, 0] = 0.5
    if kind == "diag":  # draws from the target itself, around its mean
        q = (otgt.mean + otgt.scale * rs.standard_normal((C, D))).astype(F)
    return q


@pytest.mark.parametrize("kind, D, sigma_kind, mode, correct, inplace", CASES)
def test_single_transition_matches_oracle(kind, D, sigma_kind, mode, correct, inplace):
    rs = np.random.default_rng(D + 7 * len(mode) + len(kind))
    C = 256 if D <= 1024 else 32
    tgt, otgt = make_target(kind, D, rs)
    q = start(kind, D, C, rs, otgt)
    ind = mode in ("rmh_ind", "irmh")  # an independent proposal about as wide as the chains, centred on them
    sigma = make_sigma(sigma_kind, D, 0.7 if ind else 2.4 / np.sqrt(D), rs)
    mean = q.mean(0).astype(F) if ind else None
    keys = oprng.split(oprng.key(D + len(mode)), C)
    new, info, before = run_step(tgt, q, keys, mode, sigma, mean, correct, inplace)
    acc, _ = compare(keys, q, otgt, mode, sigma, mean, correct, new, info, before)
    if D <= 1024 and mode in ("additive", "rmh"):  # the step sizes keep both outcomes in play
        assert 0 < acc.mean() < 1


def test_hier_logit_10000_matches_oracle():
    C, D = 8, 10000
    x, bits = bj.targets.HierLogit.synthetic_data(D - 4, seed=1)
    tgt, otgt = bj.targets.HierLogit(x, bits), otargets.HierLogit(x, bits)
    rs = np.random.default_rng(3)
    q = (0.3 * rs.standard_normal((C, D))).astype(F)
    for mode, correct in (("additive", False), ("irmh", True)):
        sigma = np.full(D, 0.002, F)
        mean = q.mean(0).astype(F) if mode == "irmh" else None
        keys = oprng.split(oprng.key(4 + len(mode)), C)
        new, info, before = run_step(tgt, q, keys, mode, sigma, mean, correct)
        compare(keys, q, otgt, mode, sigma, mean, correct, new, info, before)


@pytest.mark.parametrize("src, D", [("diag_gaussian", 100), ("diag_gaussian_big", 2048)])
def test_plugin_single_transition_matches_oracle(src, D):
    from blackjax_b200 import plugin
    rs = np.random.default_rng(D)
    C = 128 if D <= 1024 else 16
    tgt = bj.targets.UserTarget(D, plugin.read_example(src), np.ones(D, F), name=src)
    otgt = otargets.StdNormal(D)
    q = (0.7 * rs.standard_normal((C, D))).astype(F)
    for mode, inplace in (("additive", False), ("irmh", True)):
        sigma = np.full(D, 2.4 / np.sqrt(D), F) if mode == "additive" else np.full(D, 0.7, F)
        mean = np.zeros(D, F) if mode == "irmh" else None
        keys = oprng.split(oprng.key(7), C)
        new, info, before = run_step(tgt, q, keys, mode, sigma, mean, mode == "irmh", inplace)
        compare(keys, q, otgt, mode, sigma, mean, mode == "irmh", new, info, before)


def test_bounded_gaussian_nan_candidates_are_rejected():
    """The box at +-2 gives NaN log-densities outside: those candidates are rejected with acceptance rate 0 (NaN maps to
    -inf), their chains keep their state bit for bit, and no chain leaves the box."""
    from blackjax_b200 import plugin
    D, C, B = 2, 4096, 2.0
    tgt = bj.targets.UserTarget(D, plugin.read_example("bounded_gaussian"), np.array([B], F), name="bounded_gaussian")
    otgt = otargets.BoundedGaussian(D, B)
    rs = np.random.default_rng(2)
    q = rs.uniform(-1.5, 1.5, (C, D)).astype(F)
    keys = oprng.split(oprng.key(8), C)
    for inplace in (False, True):
        new, info, before = run_step(tgt, q, keys, "additive", F(1.5), None, False, inplace)
        acc, oi = compare(keys, q, otgt, "additive", F(1.5), None, False, new, info, before)
        nan = np.isnan(oi["candidate"][1])
        assert nan.sum() > C // 10
        assert not acc[nan].any() and (npy(info.acceptance_rate)[nan] == 0).all()
        np.testing.assert_array_equal(npy(new.position)[nan], q[nan])
    _, hist, _ = bj.sample_random_walk_native(tk(oprng.key(3)), rw.init(tf(q), tgt), tgt, 50, proposal=rw.normal(1.5))
    assert torch.all(hist.abs() < B)


def test_plugins_bit_identical_to_builtin():
    from blackjax_b200 import plugin
    for D, src in ((100, "diag_gaussian"), (2048, "diag_gaussian_big")):
        C = 32
        user = bj.targets.UserTarget(D, plugin.read_example(src), np.ones(D, F), name=src)
        builtin = bj.targets.StdNormal(D)
        q = tf(np.random.default_rng(D).standard_normal((C, D)).astype(F))
        key = tk(oprng.key(5))
        for prop, corr in ((rw.normal(0.1), None), (rw.gaussian_distribution(0.0, 1.0), rw.gaussian_logdensity(0.0, 1.0))):
            a = bj.sample_random_walk_native(key, rw.init(q.clone(), builtin), builtin, 6, proposal=prop,
                                             proposal_logdensity_fn=corr)
            b = bj.sample_random_walk_native(key, rw.init(q.clone(), user), user, 6, proposal=prop,
                                             proposal_logdensity_fn=corr)
            assert torch.equal(a[0].position, b[0].position) and torch.equal(a[0].logdensity, b[0].logdensity)
            assert torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])


def stepwise(key, st, tgt, mode, sigma, mean, correct, T_, thin, chain_offset):
    build, prop, corr = descriptors(mode, sigma, mean, correct)
    kern = build(chain_offset=chain_offset)
    hist, acc = [], []
    for t, k in enumerate(oprng.split(key, T_)):
        st, info = kern(tk(k), st, tgt, prop) if corr is None else kern(tk(k), st, tgt, prop, corr)
        acc.append(npy(info.acceptance_rate))
        if (t + 1) % thin == 0:
            hist.append(npy(st.position))
    return st, np.stack(hist), np.stack(acc), prop, corr


@pytest.mark.parametrize("D, sigma_kind, mode, correct", [(100, "vec", "irmh", True), (100, "scalar", "additive", False),
                                                          (64, "dense", "additive", False),
                                                          (64, "dense", "rmh_ind", False),
                                                          (2048, "vec", "rmh_ind", True), (2048, "scalar", "rmh", False)])
def test_native_loop_bit_identical_to_steps(D, sigma_kind, mode, correct):
    rs = np.random.default_rng(5)
    C, T_, thin, off = 40, 10, 2, 7
    tgt, _ = make_target("std", D, rs)
    sigma = make_sigma(sigma_kind, D, 1.0 if mode in ("irmh", "rmh_ind") else 2.4 / np.sqrt(D), rs)
    sigma = sigma if np.ndim(sigma) == 0 else tf(sigma)
    mean = tf(np.full(D, 0.1, F)) if mode in ("irmh", "rmh_ind") else None
    q = tf((0.8 * rs.standard_normal((C, D))).astype(F))
    key = oprng.key(21)
    st0 = rw.init(q, tgt)
    ref, h_ref, a_ref, prop, corr = stepwise(key, st0, tgt, mode, sigma, mean, correct, T_, thin, off)
    fin, hist, acc = bj.sample_random_walk_native(tk(key), st0, tgt, T_, proposal=prop, proposal_logdensity_fn=corr,
                                                  thin=thin, chain_offset=off)
    np.testing.assert_array_equal(npy(fin.position), npy(ref.position))
    np.testing.assert_array_equal(npy(fin.logdensity), npy(ref.logdensity))
    np.testing.assert_array_equal(npy(hist), h_ref)
    np.testing.assert_array_equal(npy(acc), a_ref)
    assert 0 < a_ref.mean() < 1


@pytest.mark.parametrize("D", [96, 2048])
def test_chain_offset_matches_explicit_per_chain_keys(D):
    """A shared step key folded with chain_offset + c is the chain's key: the same draws as explicit per-chain keys
    fold_in(step_key, chain_offset + c), and as one handle over all chains."""
    rs = np.random.default_rng(8)
    C = 64
    tgt = bj.targets.StdNormal(D)
    q = tf((0.5 * rs.standard_normal((C, D))).astype(F))
    key = oprng.key(3)
    prop = rw.normal(1.0 / np.sqrt(D))
    whole = bj.sample_random_walk_native(tk(key), rw.init(q, tgt), tgt, 6, proposal=prop)
    kern = rw.build_additive_step()
    for lo in (0, 32):
        part = bj.sample_random_walk_native(tk(key), rw.init(q[lo:lo + 32].clone(), tgt), tgt, 6, proposal=prop,
                                            chain_offset=lo)
        assert torch.equal(part[0].position, whole[0].position[lo:lo + 32])
        assert torch.equal(part[1], whole[1][:, lo:lo + 32]) and torch.equal(part[2], whole[2][:, lo:lo + 32])
        st = rw.init(q[lo:lo + 32].clone(), tgt)
        for k in oprng.split(key, 6):
            st, _ = kern(tk(oprng.fold_in(k, np.arange(lo, lo + 32))), st, tgt, prop)
        assert torch.equal(st.position, part[0].position)


NORMAL_1_2 = bj.targets.DiagGaussian(np.array([2.0]), mean=np.array([1.0], F))


@pytest.mark.parametrize("name", ["random_walk", "rmh", "irmh"])
def test_univariate_normal(name):
    """test_sampling.py test_random_walk / test_rmh / test_irmh, through the top-level API."""
    tgt = NORMAL_1_2
    if name == "random_walk":
        alg = bj.additive_step_random_walk.normal_random_walk(tgt, sigma=np.array([1.0], F))
    elif name == "rmh":
        alg = bj.rmh(tgt, proposal_generator=rw.gaussian_proposal(25.0))
    else:
        alg = bj.irmh(tgt, proposal_distribution=rw.gaussian_distribution(1.0, 25.0))
    C, T_, burn = 2048, 300, 100
    st = alg.init(tf(np.ones((C, 1), F)))
    keys = oprng.split(oprng.key(0), T_)
    draws = []
    for t in range(T_):
        st, info = alg.step(tk(keys[t]), st)
        if t >= burn:
            draws.append(st.position)
    s = torch.stack(draws).double()
    np.testing.assert_allclose(s.mean().item(), 1.0, rtol=1e-1)
    np.testing.assert_allclose(s.var().item(), 4.0, rtol=1e-1)


def var_z(hist, var, tgt):
    """(sample variance of all draws, |its error| / MCSE) for a zero-mean scalar chain history [T, C, 1]."""
    from blackjax_b200.diagnostics import effective_sample_size
    d2 = hist.double() ** 2
    ess = effective_sample_size(d2.float().contiguous(), tgt).double()
    v = d2.mean().item()
    return v, abs(v - var) / (d2.std().item() / ess.sqrt().item())


def test_correction_removes_the_independent_proposal_bias():
    """N(0, 1) with the independent proposal N(0, 2^2): irmh with gaussian_logdensity gives variance 1 within 5 MCSE;
    without it the stationary law is N(0, 0.8) (the target times the proposal density), and the bias shows."""
    C, T_, burn = 8192, 400, 50
    tgt = bj.targets.StdNormal(1)
    q = tf(np.zeros((C, 1), F))
    prop = rw.gaussian_distribution(0.0, 2.0)
    _, h, _ = bj.sample_random_walk_native(tk(oprng.key(1)), rw.init(q, tgt), tgt, T_, proposal=prop,
                                           proposal_logdensity_fn=rw.gaussian_logdensity(0.0, 2.0))
    v, z = var_z(h[burn:], 1.0, tgt)
    assert z < 5, (v, z)
    _, h, _ = bj.sample_random_walk_native(tk(oprng.key(1)), rw.init(q, tgt), tgt, T_, proposal=prop)
    v, z = var_z(h[burn:], 1.0, tgt)
    assert z > 20, (v, z)
    v, z = var_z(h[burn:], 0.8, tgt)
    assert z < 5, (v, z)


def test_readme_loop():
    """The reference README loop, unchanged except for the descriptors."""
    tgt = bj.targets.StdNormal(4)
    position = tf(np.zeros((8, 4), F))
    key = tk(oprng.key(0))
    for alg in (bj.additive_step_random_walk.normal_random_walk(tgt, 0.5),
                bj.rmh(tgt, rw.gaussian_proposal(0.5)),
                bj.irmh(tgt, rw.gaussian_distribution(0.0, 1.0), rw.gaussian_logdensity(0.0, 1.0))):
        state = alg.init(position)
        state, info = alg.step(key, state)
        assert state.position.shape == (8, 4) and info.is_accepted.dtype == torch.bool
        assert info.proposal is state


def test_stored_logdensity_used_as_given():
    """RWState(position, logdensity=1.0): the stored value, not the target's, enters the acceptance ratio."""
    tgt = bj.targets.StdNormal(1)
    q = tf(np.zeros((64, 1), F))
    keys = oprng.split(oprng.key(6), 64)
    _, info = rw.build_additive_step()(tk(keys), rw.RWState(q, 1.0), tgt, rw.normal(0.5))
    _, oi = orw.step(keys, np.zeros((64, 1), F), F(1.0), otargets.StdNormal(1), sigma=F(0.5))
    close(npy(info.acceptance_rate), oi["acceptance_rate"], scale=1.0)


def test_rejections():
    from blackjax_b200._engine import get_engine
    C = 4
    k = tk(oprng.split(oprng.key(0), C))
    tgt = bj.targets.StdNormal(8)
    st = rw.init(tf(np.zeros((C, 8), F)), tgt)
    eng = get_engine(st.position, tgt)
    with pytest.raises(_lib.BjxError, match="needs a proposal: call bjx_set_rw_proposal"):
        eng.rw_step(k, *st)
    eng.ensure_rw_proposal(_lib.RW_ADDITIVE, 1.0)
    with pytest.raises(_lib.BjxError, match="position-independent proposal"):
        eng.rw_step(k, *st, correct=True)
    eng.ensure_rw_proposal(_lib.RW_INDEPENDENT, tf(np.eye(8, dtype=F)), 0.0)
    with pytest.raises(_lib.BjxError, match="not built for a dense sigma"):
        eng.rw_step(k, *st, correct=True)
    eng.rw_step(k, *st)  # the dense sigma without the correction runs
    D = 132  # a dense sigma beyond 128 dims
    tgt = bj.targets.StdNormal(D)
    st = rw.init(tf(np.zeros((C, D), F)), tgt)
    with pytest.raises(_lib.BjxError, match="dense random-walk sigma is built for dim <= 128"):
        rw.build_additive_step()(k, st, tgt, rw.normal(tf(np.eye(D, dtype=F))))
    D = 256  # the tensor-core dense target path
    A = np.random.default_rng(1).standard_normal((D, D))
    tgt = bj.targets.DenseGaussian(A @ A.T / D + np.eye(D))
    st = rw.init(tf(np.zeros((C, D), F)), tgt)
    with pytest.raises(_lib.BjxError, match="tensor-core dense target path"):
        rw.build_rmh()(k, st, tgt, rw.gaussian_proposal(0.1))
