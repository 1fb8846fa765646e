"""MALA and Barker's proposal on the GPU: one teacher-forced transition against the float32 oracles (oracle/mala.py,
oracle/barker.py) over the row size classes and the big rows, the native loops bit-identical to step calls, and the
rejections.  Barker's signs may differ from the oracle only where its margin is below 1e-5 * 64, accept decisions only
where u lies within that of the oracle's acceptance probability or between the two probabilities."""
import numpy as np
import pytest
import torch

import blackjax_b200 as bj
from blackjax_b200 import _lib
from oracle import barker as ob
from oracle import mala as om
from oracle import prng as oprng
from test_gpu_parity import close, make_target, npy, tf, tk

pytestmark = pytest.mark.gpu
F = np.float32
TIE = 1e-5 * 64


def run_step(sampler, tgt, q, eps, keys, imm):
    """One transition through Engine.langevin_step with every bjx_langevin_info field."""
    from blackjax_b200._engine import get_engine
    from blackjax_b200.mcmc import barker
    st = bj.mala.init(tf(q), tgt)
    eng = get_engine(st.position, tgt)
    if sampler == "barker":
        barker.install_metric(eng, imm)
    C, D = q.shape
    f = dict(acceptance_rate=torch.empty(C, device="cuda"), is_accepted=torch.empty(C, dtype=torch.uint8, device="cuda"),
             proposal_position=torch.empty(C, D, device="cuda"), proposal_logdensity=torch.empty(C, device="cuda"),
             proposal_grad=torch.empty(C, D, device="cuda"))
    init = (npy(st.logdensity), npy(st.logdensity_grad))
    qo, lo, go = eng.langevin_step(sampler, tk(keys), *st, eps, info_fields=f)
    torch.cuda.synchronize()
    f = {k: npy(v) for k, v in f.items()}
    f["init"] = init  # the oracle starts from the same state (teacher forcing)
    return (npy(qo), npy(lo), npy(go)), f


def start(kind, tgt_o, C, D, rs):
    """Chains near the target, so that the transitions accept at a moderate rate."""
    if kind == "diag":
        return (tgt_o.mean + tgt_o.scale * rs.standard_normal((C, D))).astype(F)
    if kind == "funnel":
        q = rs.standard_normal((C, D)).astype(F)
        q[:, 0] = 0.0
        return q
    return (0.5 * rs.standard_normal((C, D))).astype(F)


CASES = [("mala", "std", 1, "none"), ("mala", "diag", 18, "none"), ("mala", "funnel", 128, "none"),
         ("mala", "diag", 1024, "none"), ("mala", "funnel", 2048, "none"), ("mala", "dense", 100, "none"),
         ("mala", "diag", 1028, "none"),
         ("barker", "std", 2, "diag"), ("barker", "diag", 100, "per_chain"), ("barker", "funnel", 512, "diag"),
         ("barker", "diag", 128, "dense"), ("barker", "dense", 18, "dense"), ("barker", "diag", 1028, "diag"),
         ("barker", "funnel", 2048, "per_chain"), ("barker", "std", 1024, "per_chain"),
         # the CTA rows past the 14-slot leapfrog edge and at the 3-row kernels' 18432 dims (221 664 B of shared memory)
         ("mala", "diag", 10756, "none"), ("mala", "funnel", 18432, "none"),
         ("barker", "funnel", 10756, "per_chain"), ("barker", "diag", 18432, "diag")]
# the hierarchical logistic regression on the CTA rows: (D, through the hier_logit_big plug-in)
HIER_LANGEVIN = [(10000, False), (18432, False), (18432, True)]


def close_grad(a, b, kind, D):
    """The funnel's neck component is a sum of D terms that cancel: it is held to rtol times D."""
    if kind == "funnel":
        close(a[:, 1:], b[:, 1:])
        close(a[:, 0], b[:, 0], scale=float(D))
    else:
        close(a, b)


def compare(sampler, keys, q, otgt, eps, imm, got, ginfo, D, kind):
    lq, gq = ginfo["init"]
    if sampler == "mala":
        (oq, ol, og), oi = om.step(keys, q, lq, gq, otgt, eps)
        ok = np.ones(q.shape[0], bool)
    else:
        (oq, ol, og), oi = ob.step(keys, q, lq, gq, otgt, eps, imm)
        # a sign may differ only where its draw is a tie; such a chain's proposal differs and is left out below
        tie = oi["sign_margins"] <= TIE
        y_o, y_g = oi["proposal"][0], ginfo["proposal_position"]
        differs = ~np.isclose(y_g, y_o, rtol=1e-4, atol=1e-5)
        assert not (differs & ~tie).any()
        ok = ~differs.any(axis=-1)
    assert ok.mean() > 0.5
    y, ly, gy = oi["proposal"]
    close(ginfo["proposal_position"][ok], y[ok])
    close(ginfo["proposal_logdensity"][ok], ly[ok], scale=np.abs(ly[ok]).max() + D)
    close_grad(ginfo["proposal_grad"][ok], gy[ok], kind, D)
    acc = ginfo["is_accepted"].astype(bool)
    same = acc == oi["is_accepted"]
    # p = exp(log_p_accept), a difference of sums whose terms are the size of the log-densities
    close(ginfo["acceptance_rate"][ok], oi["acceptance_rate"][ok], scale=1.0 + np.abs(lq).max())
    # a decision may differ only where u lies within TIE of the oracle's p or between the two p's (rows of ~1e4 dims have
    # log-densities of ~1e4, whose rounding p carries)
    dp = np.abs(ginfo["acceptance_rate"] - oi["acceptance_rate"])
    assert np.all(same | (oi["margin"] <= np.maximum(TIE, dp)) | ~ok)
    keep = same & ok
    close(got[0][keep], oq[keep])
    close_grad(got[2][keep], og[keep], kind, D)
    return acc


@pytest.mark.parametrize("sampler, kind, D, metric", CASES)
@pytest.mark.parametrize("pce", [False, True])
def test_single_transition_matches_oracle(sampler, kind, D, metric, pce):
    rs = np.random.default_rng(D + (7 if pce else 0))
    C = 64
    tgt, otgt = make_target(kind, D, rs)
    q = start(kind, otgt, C, D, rs)
    base = (0.25 if sampler == "mala" else 1.2) * D ** (-1.0 / 3) * (0.4 if kind in ("diag", "dense") else 1.0)
    base *= 0.2 if (sampler == "mala" and kind == "diag") else 1.0
    base *= 0.05 if (sampler == "mala" and kind == "funnel" and D > 10000) else 1.0   # the neck stiffens with D
    eps = (base * (0.5 + 0.5 * rs.uniform(size=C))).astype(F) if pce else F(base)
    imm = None
    if metric == "diag":
        imm = np.exp(rs.uniform(-0.5, 0.5, D)).astype(F)
    elif metric == "per_chain":
        imm = np.exp(rs.uniform(-0.5, 0.5, (C, D))).astype(F)
    elif metric == "dense":
        A = rs.standard_normal((D, D))
        imm = (A @ A.T / D + np.eye(D)).astype(F)
    keys = oprng.split(oprng.key(D), C)
    got, ginfo = run_step(sampler, tgt, q, tf(eps) if pce else float(eps), keys, None if imm is None else tf(imm))
    acc = compare(sampler, keys, q, otgt, eps, imm, got, ginfo, D, kind)
    assert acc.any()  # the step sizes give some acceptances: the comparison covers accepted proposals


@pytest.mark.parametrize("sampler", ["mala", "barker"])
def test_hier_logit_10000_matches_oracle(sampler):
    """BASELINE config 5's hierarchical logistic regression on the CTA rows, teacher-forced: at D = 10000, at the 3-row
    kernels' 18432 dims, and there through the hier_logit_big plug-in."""
    from blackjax_b200 import plugin
    from oracle import targets as otargets
    C = 6
    for D, user in HIER_LANGEVIN:
        G = D - 4
        x, bits = bj.targets.HierLogit.synthetic_data(G, seed=1)
        tgt, otgt = bj.targets.HierLogit(x, bits), otargets.HierLogit(x, bits)
        if user:
            theta = np.concatenate([np.asarray([G, 0, 0, 0], F), x.reshape(-1).astype(F), bits.astype(F)])
            tgt = bj.targets.UserTarget(D, plugin.read_example("hier_logit_big"), theta, name="hier_logit_big")
        rs = np.random.default_rng(3)
        q = (0.3 * rs.standard_normal((C, D))).astype(F)
        imm = np.exp(rs.uniform(-0.3, 0.3, D)).astype(F) if sampler == "barker" else None
        eps = F(2e-4) if sampler == "mala" else F(2e-3)
        keys = oprng.split(oprng.key(4), C)
        got, ginfo = run_step(sampler, tgt, q, float(eps), keys, None if imm is None else tf(imm))
        compare(sampler, keys, q, otgt, eps, imm, got, ginfo, D, "hier")


def stepwise(sampler, key, st, tgt, eps, imm, T_, thin, chain_offset):
    kern = (bj.mala if sampler == "mala" else bj.barker).build_kernel(chain_offset=chain_offset)
    hist, acc = [], []
    for t, k in enumerate(oprng.split(key, T_)):
        args = (eps,) if sampler == "mala" else (eps, imm)
        st, info = kern(tk(k), st, tgt, *args)
        acc.append(npy(info.acceptance_rate))
        if (t + 1) % thin == 0:
            hist.append(npy(st.position))
    return st, np.stack(hist), np.stack(acc)


@pytest.mark.parametrize("sampler", ["mala", "barker"])
@pytest.mark.parametrize("D", [100, 2048])
def test_native_loop_bit_identical_to_steps(sampler, D):
    rs = np.random.default_rng(5)
    C, T_, thin, off = 40, 12, 3, 7
    tgt, _ = make_target("diag", D, rs)
    q = tf((0.5 * rs.standard_normal((C, D))).astype(F))
    eps = tf((0.05 + 0.1 * rs.uniform(size=C)).astype(F))
    imm = tf(np.exp(rs.uniform(-0.5, 0.5, D)).astype(F)) if sampler == "barker" else None
    key = oprng.key(21)
    st0 = bj.mala.init(q, tgt)
    ref, h_ref, a_ref = stepwise(sampler, key, st0, tgt, eps, imm, T_, thin, off)
    fn = bj.sample_mala_native if sampler == "mala" else bj.sample_barker_native
    extra = () if sampler == "mala" else (imm,)
    fin, hist, acc = fn(tk(key), st0, tgt, eps, T_, *extra, thin=thin, chain_offset=off)
    np.testing.assert_array_equal(npy(fin.position), npy(ref.position))
    np.testing.assert_array_equal(npy(fin.logdensity), npy(ref.logdensity))
    np.testing.assert_array_equal(npy(fin.logdensity_grad), npy(ref.logdensity_grad))
    np.testing.assert_array_equal(npy(hist), h_ref)
    np.testing.assert_array_equal(npy(acc), a_ref)


def test_rejections():
    from blackjax_b200.mcmc import barker
    from blackjax_b200.mcmc.metrics import LowRankMetric
    D, C = 8, 4
    q = tf(np.zeros((C, D), F))
    st = bj.barker.init(q, bj.targets.StdNormal(D))
    k = tk(oprng.split(oprng.key(0), C))
    kern = barker.build_kernel()
    with pytest.raises(_lib.BjxError, match="Barker is built for diagonal"):  # per-chain dense
        kern(k, st, bj.targets.StdNormal(D), 0.1, tf(np.tile(np.eye(D, dtype=F), (C, 1, 1))))
    U = np.linalg.qr(np.random.default_rng(0).standard_normal((D, 2)))[0].astype(F)
    with pytest.raises(_lib.BjxError, match="Barker is built for diagonal"):  # low rank
        kern(k, st, bj.targets.StdNormal(D), 0.1, LowRankMetric(tf(np.ones(D, F)), tf(U), tf(np.array([2.0, 0.5], F))))
    Dd = 256
    qd = tf(np.zeros((C, Dd), F))
    std = bj.barker.init(qd, bj.targets.StdNormal(Dd))
    with pytest.raises(_lib.BjxError, match="dim <= 128"):  # dense metric on the tensor-core path
        kern(tk(oprng.split(oprng.key(0), C)), std, bj.targets.StdNormal(Dd), 0.1, tf(np.eye(Dd, dtype=F)))
    A = np.random.default_rng(1).standard_normal((Dd, Dd))
    dense_tgt = bj.targets.DenseGaussian(A @ A.T / Dd + np.eye(Dd))
    for mod in (bj.mala, bj.barker):  # dense target beyond 128 dims (tensor-core path)
        std = mod.init(qd, dense_tgt)
        args = (0.1,) if mod is bj.mala else (0.1, None)
        with pytest.raises(_lib.BjxError, match="tensor-core dense path"):
            mod.build_kernel()(tk(oprng.split(oprng.key(0), C)), std, dense_tgt, *args)


def test_plugins_match_builtin():
    """The diag_gaussian plug-in against StdNormal (rows) and diag_gaussian_big against the built-in diagonal Gaussian at
    D = 2048 (CTA rows): bit-identical native loops."""
    from blackjax_b200 import plugin
    for D, src in ((100, "diag_gaussian"), (2048, "diag_gaussian_big")):
        C = 32
        user = bj.targets.UserTarget(D, plugin.read_example(src), np.ones(D, F), name=src)
        builtin = bj.targets.StdNormal(D)
        q = tf(np.random.default_rng(D).standard_normal((C, D)).astype(F))
        key = tk(oprng.key(5))
        for sampler in ("mala", "barker"):
            fn = bj.sample_mala_native if sampler == "mala" else bj.sample_barker_native
            extra = () if sampler == "mala" else (tf(np.ones(D, F)),)
            a = fn(key, bj.mala.init(q.clone(), builtin), builtin, 0.3, 6, *extra)
            b = fn(key, bj.mala.init(q.clone(), user), user, 0.3, 6, *extra)
            assert torch.equal(a[0].position, b[0].position) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])


def test_bounded_gaussian_rejects_nan_proposals():
    """NaN log-densities outside the bound: no crash, every chain finite; MALA rejects (p = 0), Barker rejects with a
    NaN acceptance rate."""
    from blackjax_b200 import plugin
    from oracle import targets as otargets
    D, C = 2, 256
    tgt = bj.targets.UserTarget(D, plugin.read_example("bounded_gaussian"), np.array([1.0], F), name="bounded_gaussian",
                                dense_metric=False, general_integrators=True)
    otgt = otargets.BoundedGaussian(D, 1.0)
    q = (0.9 * np.random.default_rng(4).uniform(-1, 1, (C, D))).astype(F)
    keys = oprng.split(oprng.key(11), C)
    for sampler in ("mala", "barker"):
        got, gi = run_step(sampler, tgt, q, 0.5, keys, tf(np.ones(D, F)))
        assert np.isfinite(got[0]).all() and np.isfinite(got[1]).all()
        nan_prop = ~np.isfinite(gi["proposal_logdensity"])
        assert nan_prop.any() and not gi["is_accepted"].astype(bool)[nan_prop].any()
        p = gi["acceptance_rate"][nan_prop]
        assert np.all(p == 0) if sampler == "mala" else np.all(np.isnan(p))
        lq, gq = otgt(q)
        oi = (om.step(keys, q, lq, gq, otgt, 0.5) if sampler == "mala" else
              ob.step(keys, q, lq, gq, otgt, 0.5, np.ones(D, F)))[1]
        np.testing.assert_array_equal(nan_prop, ~np.isfinite(oi["proposal"][1]))


def test_barker_preconditioning():
    """A DenseGaussian with precision P under the dense metric M^-1 against precision (M^1/2)^T P M^1/2 under the
    identity metric, same keys, positions mapped by M^1/2 = chol(M^-1)^-T."""
    D, C = 6, 512
    rs = np.random.default_rng(2)
    B = rs.standard_normal((D, D))
    Pm = B @ B.T / D + np.eye(D)
    A = rs.standard_normal((D, D))
    imm = A @ A.T / D + np.eye(D)
    Ms = np.linalg.inv(np.linalg.cholesky(imm)).T
    tq, tu = bj.targets.DenseGaussian(Pm), bj.targets.DenseGaussian(Ms.T @ Pm @ Ms)
    u = rs.standard_normal((C, D))
    q = u @ Ms.T
    sq, su = bj.barker.init(tf(q), tq), bj.barker.init(tf(u), tu)
    kern = bj.barker.build_kernel()
    alive = np.ones(C, bool)  # chains whose decisions have agreed so far (they differ only on rounding ties)
    for t in range(5):
        k = tk(oprng.split(oprng.fold_in(oprng.key(6), t), C))
        sq, iq = kern(k, sq, tq, 0.8, tf(imm))
        su, iu = kern(k, su, tu, 0.8, None)
        alive &= npy(iq.is_accepted) == npy(iu.is_accepted)
        np.testing.assert_allclose(npy(sq.position)[alive], (npy(su.position) @ Ms.T)[alive], rtol=1e-3, atol=1e-3)
        np.testing.assert_allclose(npy(iq.acceptance_rate)[alive], npy(iu.acceptance_rate)[alive], rtol=1e-3,
                                   atol=1e-3)
    assert alive.mean() > 0.98 and npy(iq.is_accepted).any()


def test_barker_invariance_2d():
    """10000 chains started from N(0, I) on a 2-D standard normal: after 50 steps mean 0 and covariance I within 0.1."""
    C, D = 10000, 2
    tgt = bj.targets.StdNormal(D)
    st = bj.barker.init(tf(np.random.default_rng(8).standard_normal((C, D)).astype(F)), tgt)
    fin, _, _ = bj.sample_barker_native(tk(oprng.key(3)), st, tgt, 1.0, 50, keep_history=False)
    x = npy(fin.position).astype(np.float64)
    np.testing.assert_allclose(x.mean(0), 0.0, atol=0.1)
    np.testing.assert_allclose(np.cov(x.T), np.eye(D), atol=0.1)


@pytest.mark.parametrize("sampler, eps", [("mala", 1e-5), ("barker", 0.1)])
def test_regression_posterior(sampler, eps):
    """tests/mcmc/test_sampling.py's linear regression (scale 1, coefficient 3, 1000 points) through the LinearRegression
    plug-in: 10000 steps, the first 3000 dropped, the reference's tolerances on every chain."""
    rs = np.random.default_rng(42)
    x = rs.standard_normal((1000, 1)).astype(F)
    y = (3 * x[:, 0] + rs.standard_normal(1000)).astype(F)
    tgt = bj.targets.LinearRegression(x, y)
    C = 16
    st = bj.mala.init(tf(np.tile(np.array([1.0, 2.0], F), (C, 1))), tgt)
    fn = bj.sample_mala_native if sampler == "mala" else bj.sample_barker_native
    _, hist, _ = fn(tk(oprng.key(9)), st, tgt, eps, 10000)
    h = npy(hist[3000:]).astype(np.float64)
    for c in range(C):
        np.testing.assert_allclose(np.mean(np.exp(h[:, c, 0])), 1.0, rtol=1e-2, atol=1e-1)
        np.testing.assert_allclose(np.mean(h[:, c, 1]), 3.0, rtol=1e-2, atol=1e-1)


@pytest.mark.parametrize("sampler, eps", [("mala", 0.2), ("barker", 1.5)])
def test_univariate_normal_moments(sampler, eps):
    """test_sampling.py's univariate normal (mean 1, sd 2): moments within 5 MCSE over 2048 chains x 400 draws."""
    C, T_ = 2048, 600
    tgt = bj.targets.DiagGaussian(np.array([2.0]), mean=np.array([1.0], F))
    st = bj.mala.init(tf(np.zeros((C, 1), F)), tgt)
    fn = bj.sample_mala_native if sampler == "mala" else bj.sample_barker_native
    _, hist, _ = fn(tk(oprng.key(1)), st, tgt, eps, T_)
    x = npy(hist)[200:, :, 0].astype(np.float64)
    per_chain = x.mean(0)
    mcse = per_chain.std() / np.sqrt(C)
    assert abs(x.mean() - 1.0) < 5 * mcse
    v = ((x - 1.0) ** 2).mean(0)
    assert abs(v.mean() - 4.0) < 5 * v.std() / np.sqrt(C)
