"""GIST on the H100: teacher-forced single transitions against the oracle (oracle/gist.py) over the row size classes,
metrics, integrators and both instances; bit identity of the native loop, chain_offset halves and the plug-in; the edge
cases and rejections; and moments from many chains.

A disagreement with the oracle is allowed only on a tie: for the trajectory length the oracle's no-return dot at some step
within 1e-4 ||dtheta|| ||rho|| of 0, for the step size a compared |ell| within 1e-4 of |log a| or |log b| (the rule of
test_nuts_disagreements_sit_on_ties)."""
import numpy as np
import pytest
import torch

import blackjax_b200 as bj
from blackjax_b200 import _lib, plugin, targets as T
from blackjax_b200.mcmc import integrators as I
from oracle import gist as og
from oracle import hmc as ohmc
from oracle import prng as oprng
from oracle import targets as otargets
from test_gpu_parity import close, make_target, npy, tf, tk
from test_gpu_row_classes import make_metric

pytestmark = pytest.mark.gpu
F = np.float32
DEV = "cuda:0"
TIE = 1e-4

# (target, D, metric, integrator, per-chain step size, step size, instance options)
TL, SS = "trajectory_length", "step_size"
CASES = [
    ("banana", 2, "ones", "vv", False, 0.1, TL, dict(path_fraction=0.5)),
    ("banana", 2, "diag", "mclachlan", True, 0.1, SS, dict(criterion="symmetric")),
    ("funnel", 18, "diag", "vv", False, 0.1, TL, dict(path_fraction=0.0)),
    ("diag", 18, "per_chain", "vv", True, 0.2, SS, dict(criterion="asymmetric")),
    ("dense", 70, "dense", "vv", False, 0.1, TL, dict(path_fraction=1.0)),
    ("diag", 70, "low_rank", "mclachlan", False, 0.1, SS, dict(criterion="symmetric", num_integration_steps=2)),
    ("diag", 128, "dense", "vv", False, 0.1, SS, dict(criterion="symmetric")),
    ("dense", 128, "diag", "mclachlan", True, 0.1, TL, dict(path_fraction=0.5, max_num_steps=7)),
    ("funnel", 256, "low_rank", "vv", False, 0.05, TL, dict(path_fraction=0.5)),
    ("diag", 256, "per_chain", "vv", True, 0.1, SS, dict(criterion="asymmetric", max_search_steps=3)),
    ("diag", 512, "low_rank", "mclachlan", False, 0.05, TL, dict(path_fraction=0.5, max_num_steps=64)),
    ("funnel", 512, "diag", "vv", False, 0.05, SS, dict(criterion="symmetric")),
    ("diag", 1024, "diag", "vv", True, 0.05, TL, dict(path_fraction=0.5)),
    ("funnel", 1024, "per_chain", "mclachlan", False, 0.05, SS, dict(criterion="symmetric")),
    ("diag", 1024, "ones", "vv", False, 0.02, SS, dict(criterion="asymmetric", max_search_steps=0)),
]
COEF = {"vv": (I.velocity_verlet, ohmc.VELOCITY_VERLET), "mclachlan": (I.mclachlan, ohmc.MCLACHLAN)}


def device_kernel(instance, opts, integrator):
    if instance == TL:
        return bj.gist_trajectory_length.build_kernel(integrator, full_info=True, **opts), ()
    o = dict(opts)
    n = o.pop("num_integration_steps", 1)
    return bj.gist_step_size.build_kernel(integrator, full_info=True, **o), (n,)


@pytest.mark.parametrize("kind, D, metric, integ, pce, eps, instance, opts", CASES)
def test_single_transition_matches_oracle(kind, D, metric, integ, pce, eps, instance, opts):
    rs = np.random.default_rng(D * 5 + len(metric))
    C = 64
    tgt, otgt = make_target(kind, D, rs)
    dm, om = make_metric(metric, D, C, rs)
    q = (0.5 * rs.standard_normal((C, D))).astype(F)
    if kind == "funnel":
        q[:, 0] = rs.uniform(-1.0, 1.0, C)
    eps_np = (eps * np.exp(rs.uniform(-0.3, 0.3, C))).astype(F) if pce else F(eps)
    keys = oprng.split(oprng.key(D + 17), C)
    margins = np.full(C, np.inf)
    coef, ocoef = COEF[integ]
    onew, oinfo = og.gist_kernel(keys, ohmc.init(q, otgt), otgt, eps_np, om, instance=instance, coefficients=ocoef,
                                 margins=margins, **opts)
    kern, extra = device_kernel(instance, opts, coef)
    new, info = kern(tk(keys), bj.gist_trajectory_length.init(tf(q), tgt), tgt, tf(eps_np) if pce else float(eps_np), dm,
                     *extra)
    torch.cuda.synchronize()
    if instance == TL:
        fwd, rev, rej = info.num_steps_to_uturn_forward, info.num_steps_to_uturn_reverse, info.is_no_return_rejected
    else:
        fwd, rev, rej = info.step_index, info.reverse_step_index, info.search_exhausted
    same = ((npy(fwd) == oinfo["forward"]) & (npy(rev) == oinfo["reverse"]) & (npy(rej) == oinfo["rejected"])
            & (npy(info.num_integration_steps) == oinfo["num_integration_steps"])
            & (npy(info.is_accepted) == oinfo["is_accepted"]))
    # an acceptance decided within rounding of the uniform is a tie too
    u = oprng.uniform(oprng.split(keys, 3)[:, 2])
    tie = (margins < TIE) | (np.abs(u - oinfo["acceptance_rate"]) < 1e-5)
    print(f"{same.mean():.4f} identical; forward {np.unique(oinfo['forward'])}; accepted {oinfo['is_accepted'].mean():.2f}")
    assert (same | tie).all(), np.nonzero(~same & ~tie)
    assert same.mean() >= 0.9
    close(npy(info.momentum), oinfo["momentum"], rtol=1e-5)
    ok = same
    close(npy(new.position)[ok], onew[0][ok], rtol=1e-5)
    close(npy(new.logdensity_grad)[ok], onew[2][ok], rtol=1e-5)
    close(npy(new.logdensity)[ok], onew[1][ok], rtol=1e-5, scale=np.max(np.abs(onew[1])) + 1)
    close(npy(info.energy)[ok], oinfo["energy"][ok], rtol=1e-5, scale=np.max(np.abs(oinfo["energy"][ok]), initial=0) + D)
    close(npy(info.acceptance_rate)[ok], oinfo["acceptance_rate"][ok], rtol=1e-4, scale=1.0)
    if instance == SS:
        assert np.array_equal(npy(info.tuning_parameter.a), oinfo["a"])
        assert np.array_equal(npy(info.tuning_parameter.b), oinfo["b"])
        close(npy(info.step_size)[ok], oinfo["step_size"][ok], rtol=1e-6)
    if opts.get("max_num_steps", 1024) < 10:
        assert (oinfo["forward"] == opts["max_num_steps"]).any()   # the cap binds


@pytest.mark.parametrize("kind, D, instance, opts", [("diag", 18, TL, dict(path_fraction=0.5)),
                                                     ("funnel", 64, SS, dict(criterion="symmetric")),
                                                     ("diag", 64, TL, dict(path_fraction=0.0, max_num_steps=9)),
                                                     ("funnel", 18, SS, dict(criterion="asymmetric"))])
def test_per_chain_dense_metric_matches_oracle(kind, D, instance, opts):
    """One dense inverse mass matrix per chain [C, D, D] (D <= 64), teacher-forced chain by chain through the oracle."""
    rs = np.random.default_rng(7 * D + len(kind))
    C = 24
    tgt, otgt = make_target(kind, D, rs)
    A_ = rs.standard_normal((C, D, D))
    imm = (A_ @ A_.transpose(0, 2, 1) / D + np.eye(D)).astype(F)
    q = (0.5 * rs.standard_normal((C, D))).astype(F)
    if kind == "funnel":
        q[:, 0] = rs.uniform(-1.0, 1.0, C)
    keys = oprng.split(oprng.key(D + 3), C)
    kern, extra = device_kernel(instance, opts, I.velocity_verlet)
    new, info = kern(tk(keys), bj.gist_trajectory_length.init(tf(q), tgt), tgt, 0.1, tf(imm), *extra)
    torch.cuda.synchronize()
    if instance == TL:
        fwd, rev = npy(info.num_steps_to_uturn_forward), npy(info.num_steps_to_uturn_reverse)
    else:
        fwd, rev = npy(info.step_index), npy(info.reverse_step_index)
    same = np.zeros(C, bool)
    for c in range(C):
        margins = np.full(1, np.inf)
        onew, oinfo = og.gist_kernel(keys[c:c + 1], ohmc.init(q[c:c + 1], otgt), otgt, F(0.1), imm[c], instance=instance,
                                     margins=margins, **opts)
        close(npy(info.momentum)[c:c + 1], oinfo["momentum"], rtol=1e-5)
        u = oprng.uniform(oprng.split(keys[c:c + 1], 3)[:, 2])
        same[c] = (fwd[c] == oinfo["forward"][0] and rev[c] == oinfo["reverse"][0]
                   and npy(info.is_accepted)[c] == oinfo["is_accepted"][0])
        tie = margins[0] < TIE or abs(u[0] - oinfo["acceptance_rate"][0]) < 1e-5
        assert same[c] or tie, c
        if same[c]:
            close(npy(new.position)[c:c + 1], onew[0], rtol=2e-5)
            close(npy(info.energy)[c:c + 1], oinfo["energy"], rtol=1e-5, scale=np.abs(oinfo["energy"]).max() + D)
    assert same.mean() >= 0.9


def test_seam_reports_each_instances_tuning_parameter():
    from blackjax_b200.mcmc.composed import _seam, step_size as ss, trajectory_length as tl
    D, C = 8, 32
    tgt = T.StdNormal(D)
    st = _seam.init(tf(np.random.default_rng(0).standard_normal((C, D)).astype(F)), tgt)
    key, imm = bj.random.key(1, DEV), tf(np.ones(D, F))
    kern = _seam.build_kernel()
    _, info = kern(key, st, tgt, ss.tuning(), None, imm, 0.3)
    _, ref = ss.build_kernel()(key, st, tgt, 0.3, imm)
    assert isinstance(info.tuning_parameter, ss.StepSizeTuningParameter)
    for a, b in zip(info.tuning_parameter, ref.tuning_parameter):
        assert torch.equal(a, b)
    _, info = kern(key, st, tgt, tl.tuning(), None, imm, 0.3)
    _, ref = tl.build_kernel()(key, st, tgt, 0.3, imm)
    assert torch.equal(info.tuning_parameter, ref.tuning_parameter)


def stepwise(key, st0, tgt, eps, imm, T_, instance, thin=1, **opts):
    if instance == TL:
        kern, extra = bj.gist_trajectory_length.build_kernel(**opts), ()
    else:
        o = dict(opts)
        kern, extra = bj.gist_step_size.build_kernel(**o), ()
    keys = bj.random.split(key, T_)
    st = bj.gist_trajectory_length.init(st0.position.clone(), tgt)
    hist, acc, n_int = [], [], []
    for t in range(T_):
        st, info = kern(keys[t], st, tgt, eps, imm, *extra)
        if (t + 1) % thin == 0:
            hist.append(st.position)
        acc.append(info.acceptance_rate)
        n_int.append(info.num_integration_steps)
    return st, torch.stack(hist), torch.stack(acc), torch.stack(n_int)


@pytest.mark.parametrize("D, C, instance, thin, pce", [(18, 37, TL, 1, False), (512, 301, SS, 2, True),
                                                        (1024, 3001, TL, 3, True), (4, 130, SS, 1, False)])
def test_native_loop_bit_identical_to_steps(D, C, instance, thin, pce):
    rs = np.random.default_rng(C)
    tgt = T.Funnel(D)
    q = (0.3 * rs.standard_normal((C, D))).astype(F)
    q[:, 0] = rs.uniform(-1, 1, C)
    dm, _ = make_metric("per_chain" if pce else "diag", D, C, rs)
    eps = tf((0.1 * np.exp(rs.uniform(-0.5, 0.5, C))).astype(F)) if pce else 0.1
    key = bj.random.key(D + C, DEV)
    st0 = bj.gist_trajectory_length.init(tf(q), tgt)
    T_ = 6
    fin, hist, acc, n_int = bj.sample_gist_native(key, st0, tgt, eps, dm, T_, instance=instance, thin=thin)
    st, shist, sacc, sn = stepwise(key, st0, tgt, eps, dm, T_, instance, thin)
    assert torch.equal(n_int, sn) and torch.equal(acc, sacc) and torch.equal(hist, shist)
    assert torch.equal(fin.position, st.position) and torch.equal(fin.logdensity, st.logdensity)
    assert torch.equal(fin.logdensity_grad, st.logdensity_grad)
    again = bj.sample_gist_native(key, st0, tgt, eps, dm, T_, instance=instance, thin=thin)
    assert torch.equal(again[0].position, fin.position) and torch.equal(again[2], acc)
    if not pce:  # two chain_offset halves of one run
        h = C // 2
        halves = [bj.sample_gist_native(key, bj.gist_trajectory_length.init(tf(q[a:b]), tgt), tgt, eps, dm, T_,
                                        instance=instance, thin=thin, chain_offset=a)
                  for a, b in ((0, h), (h, C))]
        assert torch.equal(torch.cat([x[0].position for x in halves]), fin.position)
        assert torch.equal(torch.cat([x[2] for x in halves], 1), acc)


def test_plugin_matches_builtin():
    D, C = 100, 128
    rs = np.random.default_rng(3)
    s = np.exp(rs.uniform(-1, 1, D))
    inv_var = (1.0 / (s * s)).astype(F)   # as targets.DiagGaussian forms it
    user = T.UserTarget(D, plugin.read_example("diag_gaussian"), inv_var, name="diag_gaussian", dense_metric=True,
                        general_integrators=True)
    builtin = T.DiagGaussian(s)
    q = tf(rs.standard_normal((C, D)).astype(F))
    key = bj.random.key(9, DEV)
    for instance in (TL, SS):
        a = bj.sample_gist_native(key, bj.gist_trajectory_length.init(q.clone(), builtin), builtin, 0.2, tf(np.ones(D, F)),
                                  5, instance=instance)
        b = bj.sample_gist_native(key, bj.gist_trajectory_length.init(q.clone(), user), user, 0.2, tf(np.ones(D, F)), 5,
                                  instance=instance)
        assert torch.equal(a[0].position, b[0].position) and torch.equal(a[2], b[2]) and torch.equal(a[3], b[3])


def test_bounded_gaussian_edges():
    """NaN log-densities outside the bound: no crash, every chain finite, and a NaN proposal energy rejects."""
    D, C = 2, 256
    tgt = T.UserTarget(D, plugin.read_example("bounded_gaussian"), np.array([1.0], F), name="bounded_gaussian",
                       dense_metric=False, general_integrators=True)
    otgt = otargets.BoundedGaussian(D, 1.0)
    rs = np.random.default_rng(4)
    q = (0.5 * rs.uniform(-1, 1, (C, D))).astype(F)
    keys = oprng.split(oprng.key(11), C)
    for instance, kern in ((TL, bj.gist_trajectory_length.build_kernel()), (SS, bj.gist_step_size.build_kernel())):
        new, info = kern(tk(keys), bj.gist_trajectory_length.init(tf(q), tgt), tgt, 0.5, tf(np.ones(D, F)))
        torch.cuda.synchronize()
        onew, oinfo = og.gist_kernel(keys, ohmc.init(q, otgt), otgt, F(0.5), np.ones(D, F), instance=instance)
        assert np.isfinite(npy(new.position)).all() and np.isfinite(npy(new.logdensity)).all()
        nan_prop = ~np.isfinite(oinfo["energy"])
        assert not npy(info.is_accepted)[nan_prop].any()


def test_rejections():
    rs = np.random.default_rng(0)
    for D in (1028, 2048):
        tgt = T.StdNormal(D)
        st = bj.gist_trajectory_length.init(tf(rs.standard_normal((4, D)).astype(F)), tgt)
        with pytest.raises(_lib.BjxError, match="dim <= 1024"):
            bj.gist_trajectory_length.build_kernel()(bj.random.key(0, DEV), st, tgt, 0.1, tf(np.ones(D, F)))
    D = 256
    tgt = T.StdNormal(D)
    st = bj.gist_trajectory_length.init(tf(rs.standard_normal((4, D)).astype(F)), tgt)
    with pytest.raises(_lib.BjxError, match="tensor-core dense path"):
        bj.gist_step_size.build_kernel()(bj.random.key(0, DEV), st, tgt, 0.1, tf(np.eye(D, dtype=F)))
    imm = tf(np.ones(D, F))
    key = bj.random.key(0, DEV)
    for instance, opts in ((TL, dict(max_num_steps=0)), (TL, dict(path_fraction=1.5)), (TL, dict(path_fraction=-0.1)),
                           (SS, dict(num_integration_steps=0)), (SS, dict(max_search_steps=-1))):
        with pytest.raises(_lib.BjxError, match="libbjx error -1"):
            bj.sample_gist_native(key, st, tgt, 0.1, imm, 2, instance=instance, **opts)
    params = _lib.GistParams()
    params.instance, params.criterion, params.num_integration_steps = _lib.GIST_STEP_SIZE, 7, 1
    eng = bj._engine.get_engine(st.position, tgt)
    with pytest.raises(_lib.BjxError, match="criterion"):
        eng.gist_step(bj.random.key(0, DEV), *st, params, 0.1)


@pytest.mark.parametrize("case", ["isotropic", "correlated_dense", "funnel_neck"])
def test_moments_within_mcse(case):
    rs = np.random.default_rng(21)
    C, T_ = 4096, 200
    if case == "isotropic":
        D = 8
        tgt, imm, var = T.StdNormal(D), tf(np.ones(D, F)), np.ones(D)
        q = rs.standard_normal((C, D)).astype(F)
        run = dict(instance=TL, max_num_steps=1024)
        eps = 0.3
    elif case == "correlated_dense":
        D = 4
        A = rs.standard_normal((D, D))
        cov = A @ A.T / D + 0.5 * np.eye(D)
        tgt, imm, var = T.DenseGaussian(np.linalg.inv(cov)), tf(cov.astype(F)), np.diag(cov)
        q = (rs.standard_normal((C, D)) @ np.linalg.cholesky(cov).T).astype(F)
        run = dict(instance=SS, num_integration_steps=2)
        eps = 0.4
    else:
        D = 4
        tgt, imm, var = T.Funnel(D), tf(np.ones(D, F)), None
        y = 3.0 * rs.standard_normal(C)   # exact draws: y ~ N(0, 3^2), x_i | y ~ N(0, e^y)
        q = np.concatenate([y[:, None], np.exp(y / 2)[:, None] * rs.standard_normal((C, D - 1))], 1).astype(F)
        run = dict(instance=TL, max_num_steps=128)
        eps = 0.2
    st0 = bj.gist_trajectory_length.init(tf(q), tgt)
    fin, hist, acc, _ = bj.sample_gist_native(bj.random.key(5, DEV), st0, tgt, eps, imm, T_, **run)
    x = hist[T_ // 4:]
    ess = npy(bj.diagnostics.effective_sample_size(x.contiguous(), tgt))
    m = npy(x.mean((0, 1)))
    v = npy(x.var((0, 1)))
    if case == "funnel_neck":  # the neck y ~ N(0, 3^2)
        assert abs(m[0]) < 5 * 3.0 / np.sqrt(ess[0])
        assert abs(v[0] / 9.0 - 1) < 5 * np.sqrt(2.0 / ess[0])
    else:
        assert (np.abs(m) < 5 * np.sqrt(var / ess)).all(), (m, ess)
        assert (np.abs(v / var - 1) < 5 * np.sqrt(2.0 / ess)).all(), (v, ess)
    assert float(acc.mean()) > 0.3
