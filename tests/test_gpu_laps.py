"""LAPS on the GPU (bjx_laps_*, k_laps_burn_in) against the NumPy restatement in oracle/laps.py:
initialisation, teacher-forced burn-in steps and their ensemble update, equipartition_fullrank, bit identity (chunk size,
diagnostics, repeated runs), the adjusted phase against bjx_adjusted_mclmc_step and the bisection, the phase-boundary
choices, a recovery test on a badly scaled Gaussian and the rejections."""
import math

import numpy as np
import pytest
import torch

import blackjax_b200 as bj
from blackjax_b200 import _engine, _lib, plugin, targets as T
from blackjax_b200.adaptation import laps as L
from blackjax_b200.adaptation import laps_burn_in as lb
from blackjax_b200.mcmc import integrators
from oracle import laps as ol
from oracle import prng as oprng
from oracle import targets as otargets
from test_gpu_parity import close, npy, tf, tk

pytestmark = pytest.mark.gpu
F = np.float32


def _rel(a, b, rtol):
    a, b = float(a), float(b)
    assert (math.isnan(a) and math.isnan(b)) or a == b or abs(a - b) <= rtol * max(abs(b), 1e-30), (a, b)


def _target(name, D, rs):
    s = np.exp(rs.uniform(-0.5, 0.5, D))
    if name == "diag":
        return T.DiagGaussian(s), otargets.DiagGaussian(s)
    if name == "user":  # the diagonal Gaussian as a row plug-in, which carries k_laps_burn_in too
        inv_var = (1.0 / (np.asarray(s, np.float64) ** 2)).astype(F)
        return T.UserTarget(D, plugin.read_example("diag_gaussian"), inv_var, name="diag_gaussian"), \
            otargets.DiagGaussian(s)
    return T.Funnel(D), otargets.Funnel(D)


def _setup(name, N, D, save_num, seed):
    rs = np.random.default_rng(seed)
    tgt, otgt = _target(name, D, rs)
    q = (rs.standard_normal((N, D)) * (0.3 if name == "funnel" else 1.0) + 0.5).astype(F)
    eng = _engine.get_engine(tf(q), tgt)
    eng.set_integrator(integrators.velocity_verlet)
    adap = lb.new_state(eng, save_num, True)
    st = lb.initialize(eng, tf(q), adap, save_num)
    return eng, tgt, otgt, q, adap, st


@pytest.mark.parametrize("N, D", [(7, 100), (300, 2), (4096, 64)])
def test_initialisation_matches_oracle(N, D):
    eng, _, otgt, q, adap, st = _setup("diag", N, D, 3, N + D)
    (oq, ou, ologp, og), _ = ol.initialize(q, otgt)
    close(npy(st[1]), ou, scale=1.0 / math.sqrt(D))
    close(npy(st[3]), og)
    close(npy(st[2]), ologp, scale=float(np.max(np.abs(ologp))))
    h = lb.header(adap)
    assert h["L"] == math.inf and h["step_size"] == F(F(0.01) * np.sqrt(F(D))) and h["step_count"] == 0


# Fields held to 1e-5 relative.  Three are differences of nearly equal float32 numbers and carry an absolute rounding
# error instead: EEVPD = (E[E^2] - E[E]^2) / D on the scale of E[E^2] / D, r_max and r_avg = E[h^2] / E[h]^2 - 1 to a
# few float32 ulps of 1; equi_full is held to 1e-4 of its float64 value.
_EXACT = ("L", "step_size", "EEVPD_wanted", "equi_diag", "entropy")


@pytest.mark.parametrize("name, N, D, steps", [("diag", 1, 100, 5), ("diag", 7, 2, 5), ("diag", 7, 512, 5),
                                               ("funnel", 7, 100, 5), ("user", 7, 100, 5), ("diag", 4096, 100, 5),
                                               ("diag", 7, 1024, 5), ("diag", 4096, 1024, 3), ("diag", 64, 100, 50)])
def test_burn_in_steps_teacher_forced(name, N, D, steps):
    """Every step starts from the device's previous state: the transition within close() of the oracle's, nonans
    identical, and the ensemble update (info row, L, step size, metric, history) against the oracle's update.  The
    50-step case wraps the 3-row history many times."""
    save_num = 3
    eng, tgt, otgt, q, adap, st = _setup(name, N, D, save_num, 7 * N + D)
    cfg = lb.config(save_num, early_stop=False)
    info = torch.zeros(steps, 9, device="cuda")
    ad = ol.BurnIn(D, save_num)
    pk = oprng.key(99)
    for t in range(steps):
        prev = tuple(npy(x) for x in st)
        h0 = lb.header(adap)
        ad.L, ad.eps = F(h0["L"]), F(h0["step_size"])
        keys = ol.sampling_keys(pk, N, steps, t)
        lb.burn_in_step_(eng, tk(pk), t, steps, st, adap, cfg, info)
        new, oinfo = ol.burn_in_kernel(keys, prev, otgt, ad.L, ad.eps)
        dev = tuple(npy(x) for x in st)
        close(dev[0], new[0])
        close(dev[1], new[1], scale=1.0 / math.sqrt(D))
        close(dev[2], new[2], scale=max(float(np.max(np.abs(new[2]))), 1.0))
        close(dev[3], new[3])
        # the energy change is a float32 cancellation of log-densities (|logp| >> |E| at small step sizes): the update is
        # fed with the device transition's own, from k_mclmc_transition on the same keys (the body k_laps_burn_in runs)
        ec = torch.empty(N, device="cuda")
        nn = torch.empty(N, dtype=torch.uint8, device="cuda")
        eng.mclmc_step_(tk(keys), *(tf(x) for x in prev), float(ad.eps), float(ad.L), math.inf,
                        info_fields={"energy_change": ec, "nonans": nn})
        assert np.array_equal(npy(nn).astype(bool), oinfo.nonans)
        oinfo.energy_change = npy(ec)
        _, dinfo = ol.burn_in_kernel(keys, prev, otgt, ad.L, ad.eps)
        dinfo.energy_change = npy(ec)
        Et = ol.summaries(dev, dinfo)
        ef = ol.equi_full(dev, ol.adaptation_key(pk, t))
        row, imm = ol.update(ad, Et, 1.9, 0.1, 3, ef)
        r = npy(info[t])
        hist = npy(lb.history(adap, D, save_num))
        dev_rows = [hist[(t - j) % save_num] for j in range(min(t + 1, save_num))]
        r_scale = float(np.max(np.abs(ol.contract_history(np.stack(dev_rows), np.ones(len(dev_rows))))))
        # r = E[h^2] / E[h]^2 - 1 inherits the float32 error of the row sum sum_j h_j, its condition number times an ulp
        h64 = np.abs(np.stack(dev_rows).astype(np.float64))
        kappa = float(np.max(h64.sum(0) / np.maximum(np.abs(np.stack(dev_rows).astype(np.float64).sum(0)), 1e-300)))
        for i, k in enumerate(lb.BURN_IN_INFO):
            if k in _EXACT:
                _rel(r[i], row[k], 1e-5)
            elif k == "equi_full":
                _rel(r[i], row[k], 1e-4)
            elif k == "EEVPD":
                assert abs(r[i] - row[k]) <= 1e-5 * abs(row[k]) + 1e-4 * float(Et["Esq"]) / D + 1e-30, (r[i], row[k])
            elif t > 0:  # r_max, r_avg from the device's own history rows: a near-zero ensemble mean makes r a ratio
                # of float32 sums that the oracle's float64 means cannot reproduce (r ~ 1e6 in some dimension)
                want = ol.contract_history(np.stack(dev_rows), np.ones(len(dev_rows)))[0 if k == "r_max" else 1]
                tol = 1e-5 * abs(want) + 1e-6 * (1 + r_scale) + 4 * 2.0 ** -24 * kappa * r_scale
                assert abs(r[i] - want) <= tol, (k, r[i], want, kappa)
        h = lb.header(adap)
        _rel(h["L"], ad.L, 1e-5)
        _rel(h["step_size"], ad.eps, 1e-5)
        assert h["step_count"] == t + 1 and not h["stopped"]
        close(npy(lb.inverse_mass_matrix(adap, D)), imm, scale=float(np.max(np.abs(imm))) + 1e-6)
        # the ring: slot (t - j) % save_num holds the j-th newest row of the reference's history
        for j in range(min(t + 1, save_num)):
            close(hist[(t - j) % save_num], ad.hist[j])


def test_nan_path_keeps_the_momentum():
    N, D = 64, 2
    tgt = T.UserTarget(2, plugin.read_example("bounded_gaussian"), np.array([5.0], F), name="bounded_gaussian",
                       dense_metric=False, general_integrators=True)
    q = (0.5 * np.random.default_rng(0).standard_normal((N, D))).astype(F)
    eng = _engine.get_engine(tf(q), tgt)
    eng.set_integrator(integrators.velocity_verlet)
    adap = lb.new_state(eng, 2, True)
    st = lb.initialize(eng, tf(q), adap, 2)
    adap[lb.LS_EPS] = 100.0
    u0 = npy(st[1]).copy()
    q0 = npy(st[0]).copy()
    lb.burn_in_step_(eng, tk(oprng.key(3)), 0, 10, st, adap, lb.config(2, early_stop=False))
    bad = np.all(npy(st[0]) == q0, axis=1) & np.all(npy(st[1]) == u0, axis=1)
    assert bad.any()
    assert lb.header(adap)["step_size"] == F(50.0)


def _shifted(D):
    """A Gaussian whose ensemble mean of x is far from 0, so that the history's fluctuation r_max can fall below r_end."""
    s = np.exp(np.linspace(0, np.log(3.0), D))
    return T.DiagGaussian(s, mean=3.0 + np.linspace(0.0, 1.0, D))


def _run(tgt, N, D, T1, chunk=64, diagnostics=True, early_stop=True, seed=5):
    out = L.laps(tgt, lambda k: bj.random.normal(k, (D,)), D, T1, 300, N, None, bj.random.key(seed),
                 early_stop=early_stop, diagnostics=diagnostics, chunk=chunk)
    torch.cuda.synchronize()
    return out


def test_early_stop_chunk_size_diagnostics_and_repeat_are_bit_identical():
    N, D, T1 = 512, 64, 600
    tgt = _shifted(D)
    a = _run(tgt, N, D, T1, chunk=1)
    n1 = len(a[0]["phase_1"]["L"])
    assert 0.2 * T1 < n1 < T1  # the burn-in stopped early
    for x in (_run(tgt, N, D, T1, chunk=64), _run(tgt, N, D, T1, chunk=7), _run(tgt, N, D, T1, chunk=1)):
        for u, v in zip(a[3], x[3]):
            assert torch.equal(u, v)
        for ph in ("phase_1", "phase_2"):
            assert a[0][ph].keys() == x[0][ph].keys()
            for k in a[0][ph]:
                assert torch.equal(a[0][ph][k].nan_to_num(7.0), x[0][ph][k].nan_to_num(7.0)), (ph, k)
    c = _run(tgt, N, D, T1, chunk=64, diagnostics=False)
    assert c[0] is None
    for u, v in zip(a[3], c[3]):
        assert torch.equal(u, v)
    # the stop index is the oracle's for the device's r_max sequence, and the stopped run is the full run's prefix
    full = _run(tgt, N, D, T1, early_stop=False)
    f1 = full[0]["phase_1"]
    assert len(f1["L"]) == T1
    assert n1 == ol.stop_index(f1["r_max"].numpy(), int(np.rint(np.float32(0.2 * T1))), np.float32(0.01), T1)
    for k in a[0]["phase_1"]:
        assert torch.equal(a[0]["phase_1"][k].nan_to_num(7.0), f1[k][:n1].nan_to_num(7.0)), k


def test_adjusted_steps_are_bjx_adjusted_mclmc_step_and_the_bisection():
    N, D, S = 256, 100, 6
    rs = np.random.default_rng(2)
    tgt, otgt = _target("diag", D, rs)
    q = rs.standard_normal((N, D)).astype(F)
    eng = _engine.get_engine(tf(q), tgt)
    adap = lb.new_state(eng, 2, False)
    st = lb.initialize(eng, tf(q), adap, 2)
    imm = lb.switch_(eng, adap, True)
    eng.set_integrator(integrators.mclachlan)
    h0 = lb.header(adap)
    assert h0["bounds"] == (-math.inf, math.inf) and not h0["terminated"]
    pk = oprng.key(4)
    info = torch.zeros(S, 4, device="cuda")
    upd = ol.bisection(0.7)
    bst, eps = ((-np.inf, np.inf), False), h0["step_size"]
    for t in range(S):
        ref = [x.clone() for x in (st[0], st[2], st[3])]
        eps_dev = lb.header(adap)["step_size"]
        _rel(eps_dev, eps, 1e-5)
        lb.adjusted_step_(eng, tk(pk), t, S, (st[0], st[2], st[3]), adap, 2, 15, 0.7, True, info)
        acc = torch.empty(N, device="cuda")
        qo, lo, go = eng.adjusted_mclmc_step(tk(ol.sampling_keys(pk, N, S, t)), *ref,
                                             torch.full((N,), eps_dev, device="cuda"), 15, 1.25,
                                             info_fields={"acceptance_rate": acc})
        torch.cuda.synchronize()
        assert torch.equal(qo, st[0]) and torch.equal(go, st[3]) and torch.equal(lo, st[2])
        a_mean = float(npy(info[t])[2])
        _rel(a_mean, float(np.mean(npy(acc).astype(np.float64))), 1e-5)
        _rel(npy(info[t])[1], eps_dev, 0)
        _rel(npy(info[t])[0], F(F(eps_dev) * F(15)), 0)
        bst, eps = upd(bst, eps_dev, a_mean)
        h = lb.header(adap)
        for got, want in zip(h["bounds"], bst[0]):
            assert got == want or abs(got - want) <= 1e-5 * (1 + abs(want)), (h["bounds"], bst[0])
        assert h["terminated"] == bst[1]
    assert npy(imm).shape == (D,)


@pytest.mark.parametrize("D, want", [(100, (2, 0.7)), (256, (5, 0.9))])
def test_phase_boundary_choices(D, want):
    tgt = T.DiagGaussian(np.ones(D))
    out = L.laps(tgt, lambda k: bj.random.normal(k, (D,)), D, 20, 200, 64, None, bj.random.key(1), early_stop=False)
    assert (out[1], out[2]) == want
    assert len(out[0]["phase_2"]["L"]) == 200 // (want[0] * 15)
    out = L.laps(tgt, lambda k: bj.random.normal(k, (D,)), D, 20, 200, 64, None, bj.random.key(1), early_stop=False,
                 integrator_coefficients=integrators.velocity_verlet)
    assert (out[1], out[2]) == (1, 0.9)
    out = L.laps(tgt, lambda k: bj.random.normal(k, (D,)), D, 20, 200, 64, None, bj.random.key(1), early_stop=False,
                 acc_prob=0.8)
    assert out[2] == 0.8


def test_reference_regression_posterior():
    """tests/mcmc/test_sampling.py:743-783 on the LinearRegression plug-in: 100 chains, 1000 + 1000 steps, no early stop;
    mean(exp(log_scale)) within 0.1 of 1 and mean(coef) within 0.1 of 3."""
    rs = np.random.default_rng(42)
    x = rs.standard_normal((1000, 1)).astype(F)
    y = (3 * x[:, 0] + rs.standard_normal(1000)).astype(F)
    tgt = T.LinearRegression(x, y)
    info, gcps, acc, st = L.laps(tgt, lambda k: bj.random.normal(k, (2,)), 2, 1000, 1000, 100, None, bj.random.key(19),
                                 early_stop=False, diagonal_preconditioning=True, steps_per_sample=15, r_end=0.01)
    p = npy(st.position).astype(np.float64)
    assert (gcps, acc) == (2, 0.7) and len(info["phase_1"]["L"]) == 1000
    assert abs(np.mean(np.exp(p[:, 0])) - 1.0) < 0.1
    assert abs(np.mean(p[:, 1]) - 3.0) < 0.1


def test_badly_scaled_gaussian_is_recovered():
    N, D = 4096, 512
    s = np.exp(np.linspace(0, np.log(10.0), D))  # kappa = 100
    mean = np.linspace(-2.0, 2.0, D) * s
    tgt = T.DiagGaussian(s, mean=mean)
    info, _, _, st = L.laps(tgt, lambda k: bj.random.normal(k, (D,)), D, 500, 3000, N, None, bj.random.key(0))
    x = npy(st.position).astype(np.float64)
    mcse_m = s / np.sqrt(N)
    mcse_v = s ** 2 * np.sqrt(2.0 / N)
    assert np.all(np.abs(x.mean(0) - mean) < 5 * mcse_m)
    assert np.all(np.abs(x.var(0) - s ** 2) < 5 * mcse_v)


def test_rejections():
    D = 4
    tgt = T.DiagGaussian(np.ones(D))
    si = lambda k: bj.random.normal(k, (D,))
    key = bj.random.key(0)
    for kw, msg in [({"microcanonical": False}, "microcanonical"), ({"superchain_size": 2}, "superchain"),
                    ({"all_chains_info": lambda x: x}, "all_chains_info"), ({"contract": lambda x: 0.0}, "contract"),
                    ({"observables_for_bias": lambda x: x}, "observables")]:
        with pytest.raises(ValueError, match=msg):
            L.laps(tgt, si, D, 10, 10, 8, None, key, **kw)
    with pytest.raises(ValueError, match="mesh"):
        L.laps(tgt, si, D, 10, 10, 8, object(), key)
    with pytest.raises(ValueError, match="ndims"):
        L.laps(tgt, si, D + 1, 10, 10, 8, None, key)
    t1 = T.DiagGaussian(np.ones(1))
    with pytest.raises(_lib.BjxError, match="dim >= 2"):
        L.laps(t1, lambda k: bj.random.normal(k, (1,)), 1, 10, 10, 8, None, key)
    t2 = T.DiagGaussian(np.ones(1028))
    with pytest.raises(_lib.BjxError, match="1024"):
        L.laps(t2, lambda k: bj.random.normal(k, (1028,)), 1028, 10, 10, 8, None, key)
    P = (np.eye(132) + 0.1).astype(F)
    with pytest.raises(_lib.BjxError, match="128"):
        L.laps(T.DenseGaussian(P), lambda k: bj.random.normal(k, (132,)), 132, 10, 10, 8, None, key)
    # C ABI: one shared diagonal metric, and bias_type 2 only with equi_full
    eng, _, _, _, adap, st = _setup("diag", 8, 4, 2, 0)
    with pytest.raises(_lib.BjxError, match="bias_type 2 needs equi_full"):
        lb.burn_in_step_(eng, tk(oprng.key(1)), 0, 10, st, adap, lb.config(2, bias_type=2, equi_full=False))
    eng.set_metric(torch.ones(8, 4, device="cuda"), diagonal_only=True)
    with pytest.raises(_lib.BjxError, match="one diagonal metric"):
        lb.burn_in_step_(eng, tk(oprng.key(1)), 0, 10, st, adap, lb.config(2))
    eng._imm_key = None
