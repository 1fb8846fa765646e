"""The CTA-per-chain big-row kernels (csrc/bjx_big.cuh, csrc/bjx_big.cu; 1024 < D <= 18432) against the float32 oracle at
every dispatch edge.

One CTA owns one chain and keeps its row in shared memory.  Which compiled kernel runs depends on the target and on D:
``big_launch`` picks the leapfrog's momentum array (14 or 24 slots per thread) and ``bjx_big_hmc_step`` sends the
hierarchical logistic regression to the two-chains-per-CTA kernel up to 10240 dims.  ``kernel_for`` below restates that
table from the C++, the case lists are checked at import to reach every instance of every target at both sides of each
edge, and ``test_kernel_names_match_the_table`` pins the table to the kernels the profiler sees launched.  MALA and
Barker on these rows are compared in tests/test_gpu_langevin.py; its case lists count towards the coverage here.

Tolerances (DESIGN section 4): one step from identical inputs within 1e-5 relative, 2e-5 after five steps.  Sums of D
terms that cancel (the funnel's neck gradient, the hierarchical model's four hyper-parameter gradients) are held to rtol
times D, the size of what was summed.  An accept decision or divergence flag may differ from the oracle's only where
the oracle's energy difference sits within the measured energy disagreement of the decision boundary: the hierarchical
model's energies are ~1e5, where one float32 ulp is 0.008, and its sigmoid and softplus are MUFU approximations.
"""
import re

import numpy as np
import pytest
import torch

import blackjax_b200 as bj
from blackjax_b200 import _engine, plugin, targets as T
from oracle import adaptation as oadapt
from oracle import hmc as ohmc
from oracle import prng as oprng
from oracle import targets as otargets
from test_gpu_langevin import CASES as LANGEVIN_CASES, HIER_LANGEVIN
from test_gpu_parity import DEV, F, close, npy, tf, tk

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------------------------
# the dispatch table, restated from the C++ and checked at import
# ---------------------------------------------------------------------------------------------------------------------
BIG_THREADS = 768                                  # bjx::kBigThreads
TARGETS = ("diag", "funnel", "hier", "user_diag", "user_hier")
TK = {"diag": 0, "funnel": 1, "hier": 4, "user_diag": 5, "user_hier": 5}   # BJX_TARGET_* (include/bjx.h)
LANGEVIN_KIND = {"mala": 0, "barker": 1}           # bjx::LangevinKind


def kernel_for(target, D, op):
    """The kernel instance (demangled name without namespace, spaces or arguments) that runs ``op`` on ``target`` rows of
    D dims: bjx_big.cuh ``big_launch`` and bjx_big.cu ``bjx_big_hmc_step``."""
    tk_ = TK[target]
    if op == "init":
        return f"k_big_init<{tk_}>"
    if op in ("momentum", "energy"):
        return f"k_big_{op}"
    if op == "leapfrog":
        return f"k_big_leapfrog<{tk_},{14 if D <= 14 * BIG_THREADS else 24}>"
    if op == "hmc":
        return "k_big2_hmc_hier<512>" if target == "hier" and D <= 10240 else f"k_big_hmc<{tk_}>"
    return f"k_big_langevin<{tk_},{LANGEVIN_KIND[op]}>"


def instances(target):
    """Every big-row kernel instance a target has.  k_big_leapfrog<., 14> runs two CTAs per SM for diag and funnel, one
    for hier and the plug-ins: both occupancy variants are among the targets' instances."""
    tk_ = TK[target]
    out = {f"k_big_init<{tk_}>", "k_big_momentum", "k_big_energy", f"k_big_leapfrog<{tk_},14>",
           f"k_big_leapfrog<{tk_},24>", f"k_big_hmc<{tk_}>", f"k_big_langevin<{tk_},0>", f"k_big_langevin<{tk_},1>"}
    if target == "hier":
        out.add("k_big2_hmc_hier<512>")
    return out


# init / momentum / energy / leapfrog: (target, D, C, metric); metric "diag" (shared) or "per_chain"
BLOCK_CASES = [
    ("diag", 1028, 9, "diag"), ("diag", 2048, 40, "diag"), ("diag", 10752, 7, "per_chain"), ("diag", 10756, 5, "diag"),
    ("diag", 18432, 6, "per_chain"),
    ("funnel", 1500, 24, "diag"), ("funnel", 10752, 5, "diag"), ("funnel", 10756, 7, "per_chain"),
    ("funnel", 18432, 5, "diag"),
    ("hier", 1504, 24, "diag"), ("hier", 10000, 6, "diag"), ("hier", 10752, 5, "per_chain"), ("hier", 10756, 5, "diag"),
    ("hier", 18432, 4, "per_chain"),
    ("user_diag", 1028, 5, "diag"), ("user_diag", 10752, 5, "per_chain"), ("user_diag", 18432, 5, "diag"),
    ("user_hier", 10752, 4, "diag"), ("user_hier", 10756, 4, "per_chain"),
]
# one HMC transition at L = 0, 1, 6: (target, D, C, metric, per-chain step size, in place)
HMC_CASES = [
    ("diag", 1028, 9, "diag", False, False), ("diag", 2048, 40, "diag", False, False),
    ("diag", 10752, 7, "per_chain", True, True), ("diag", 10756, 8, "diag", True, False),
    ("diag", 18432, 6, "per_chain", False, True),
    ("funnel", 1500, 24, "diag", False, False), ("funnel", 10756, 7, "per_chain", True, False),
    ("funnel", 18432, 5, "diag", True, True),
    ("hier", 1504, 24, "diag", False, False), ("hier", 1504, 7, "per_chain", True, False),
    ("hier", 1504, 1, "per_chain", True, True), ("hier", 2052, 5, "per_chain", True, True),
    ("hier", 10000, 6, "diag", False, False),
    ("hier", 10240, 7, "per_chain", True, True),      # every thread's 20 slots full, the last CTA's second slot idles
    ("hier", 10240, 6, "diag", False, False), ("hier", 10244, 5, "per_chain", True, True),
    ("hier", 18432, 4, "diag", True, False),
    ("user_diag", 10756, 5, "per_chain", True, True), ("user_diag", 18432, 5, "diag", False, False),
    ("user_hier", 10244, 4, "diag", True, False),
]
# the native loop: (target, D, C, chain_offset)
NATIVE_CASES = [("hier", 10240, 5, 0), ("hier", 10244, 4, 0), ("diag", 18432, 6, 0), ("hier", 10240, 5, 9)]


def _reached():
    got = {t: set() for t in TARGETS}
    for t, D, _, _ in BLOCK_CASES:
        got[t] |= {kernel_for(t, D, op) for op in ("init", "momentum", "energy", "leapfrog")}
    for t, D, *_ in HMC_CASES:
        got[t].add(kernel_for(t, D, "hmc"))
    for sampler, kind, D, _ in LANGEVIN_CASES:
        if D > 1024:
            got[kind].add(kernel_for(kind, D, sampler))
    for sampler in ("mala", "barker"):
        for D, user in HIER_LANGEVIN:
            t = "user_hier" if user else "hier"
            got[t].add(kernel_for(t, D, sampler))
    return got


def _check_coverage():
    got = _reached()
    for t in TARGETS:
        if t == "user_diag":   # its Langevin kernels: test_gpu_langevin.test_plugins_match_builtin (bit-identical)
            got[t] |= {kernel_for(t, 2048, s) for s in ("mala", "barker")}
        assert got[t] == instances(t), f"{t}: cases miss {sorted(instances(t) - got[t])}"
    lf_dims = {D for _, D, _, _ in BLOCK_CASES}
    hier_hmc = {D for t, D, *_ in HMC_CASES if t == "hier"}
    assert {10752, 10756} <= lf_dims and {10240, 10244} <= hier_hmc            # both sides of both edges
    assert {1028, 18432} <= lf_dims and {1028, 18432} <= {D for _, D, *_ in HMC_CASES}
    # full and ragged last strides of each momentum array: 14 x 768 and 24 x 768 fill every thread's last slot
    for nk, lo in ((14, 1024), (24, 14 * BIG_THREADS)):
        mine = {D for D in lf_dims if lo < D <= nk * BIG_THREADS}
        assert nk * BIG_THREADS in mine and any(D % BIG_THREADS for D in mine), (nk, sorted(mine))
    assert 10240 % 512 == 0 and any(D % 512 for D in hier_hmc if D <= 10240)   # k_big2: 20 x 512 full, others ragged
    assert any(t == "hier" and D == 10240 and C % 2 and inpl for t, D, C, _, _, inpl in HMC_CASES)
    # every metric kind, step-size kind and output mode reaches the 3-row kernels and k_big2
    for kern in ("k_big_hmc", "k_big2_hmc_hier"):
        modes = {(m, p, i) for t, D, _, m, p, i in HMC_CASES if kernel_for(t, D, "hmc").startswith(kern)}
        assert {m for m, _, _ in modes} == {"diag", "per_chain"} and {p for _, p, _ in modes} == {False, True}
        assert {i for _, _, i in modes} == {False, True}


_check_coverage()


# ---------------------------------------------------------------------------------------------------------------------
# problems
# ---------------------------------------------------------------------------------------------------------------------
def big_problem(target, D, rs):
    """(device target, oracle target).  The diagonal Gaussian has a mean and a log-density offset (make_target's); the
    plug-ins take the same parameters as their built-in twins (diag_gaussian_big has neither mean nor offset)."""
    if target == "diag":
        s = np.exp(rs.uniform(-1, 1, D))
        mean = rs.standard_normal(D).astype(F)
        return T.DiagGaussian(s, mean=mean, logp_offset=0.25), otargets.DiagGaussian(s, mean=mean, logp_offset=0.25)
    if target == "funnel":
        return T.Funnel(D), otargets.Funnel(D)
    if target == "user_diag":
        s = np.exp(rs.uniform(-1, 1, D))
        user = T.UserTarget(D, plugin.read_example("diag_gaussian_big"), (1.0 / (s * s)).astype(F),
                            name="diag_gaussian_big")
        return user, otargets.DiagGaussian(s)
    G = D - 4
    x, bits = T.HierLogit.synthetic_data(G, seed=1)
    if target == "hier":
        return T.HierLogit(x, bits), otargets.HierLogit(x, bits)
    theta = np.concatenate([np.asarray([G, 0, 0, 0], F), x.reshape(-1).astype(F), bits.astype(F)])
    return T.UserTarget(D, plugin.read_example("hier_logit_big"), theta, name="hier_logit_big"), otargets.HierLogit(x, bits)


def start(target, otgt, C, D, rs):
    """Chains in the target's typical set, so that the step sizes below give a mix of accepts and rejects."""
    if target in ("diag", "user_diag"):
        mean = 0.0 if otgt.mean is None else otgt.mean
        return (mean + otgt.scale * rs.standard_normal((C, D))).astype(F)
    if target == "funnel":
        y = rs.uniform(-1, 1, C)
        q = (np.exp(y / 2)[:, None] * rs.standard_normal((C, D))).astype(F)
        q[:, 0] = y
        return q
    q = np.empty((C, D), F)
    q[:, :4] = [0.5, np.log(0.7), 1.0, -0.5]
    q[:, 4:] = 0.5 + 0.7 * rs.standard_normal((C, D - 4))
    return q


def step_size(target, D):
    """Acceptance rates between ~0.2 and 1 at L = 6 (the funnel's neck oscillates at ~sqrt(D / 2))."""
    return {"diag": 0.12, "user_diag": 0.12, "funnel": 1.4 / np.sqrt(D / 2)}.get(target, 0.007)


def make_metric(kind, C, D, rs):
    if kind == "diag":
        imm = np.exp(rs.uniform(-0.3, 0.3, D)).astype(F)
        return imm, ohmc.Metric(imm)
    imm = np.exp(rs.uniform(-0.3, 0.3, (C, D))).astype(F)
    return imm, oadapt._PerChainDiag(imm)


def neck(target):
    """Coordinates whose gradient is a sum of D terms that cancel."""
    return {"funnel": 1, "hier": 4, "user_hier": 4}.get(target, 0)


def close_row(a, b, target, D, rtol=1e-5, neck_scale=None):
    """close() per row element; the neck coordinates held to rtol * neck_scale (default D)."""
    k = neck(target)
    close(a[:, k:], b[:, k:], rtol=rtol)
    if k:
        close(a[:, :k], b[:, :k], rtol=rtol, scale=float(D if neck_scale is None else neck_scale))


def engine(tgt, C, D, imm):
    eng = _engine.Engine(DEV, C, D, tgt)
    eng.set_metric(tf(imm))
    return eng


# ---------------------------------------------------------------------------------------------------------------------
# the table against the launched kernels
# ---------------------------------------------------------------------------------------------------------------------
def _launched(fn):
    """Names (as kernel_for writes them) of the big-row kernels that fn() launches, in launch order."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    evs = sorted((e for e in prof.events() if "k_big" in e.name), key=lambda e: e.time_range.start)
    out = []
    for e in evs:
        m = re.search(r"(k_big\w*)\s*(<[^>]*>)?\s*\(", e.name)
        assert m, e.name
        out.append(m.group(1) + (m.group(2) or "").replace(" ", ""))
    return out


NAME_ROWS = [(t, D) for t in TARGETS for D in (10752, 10756, 18432)] + [("hier", 10240), ("hier", 10244)]


def test_kernel_names_match_the_table():
    """Every (target, D) row runs each operation once under the profiler; the launched kernel and its template arguments
    are the ones kernel_for predicts."""
    seen = {}
    for target, D in NAME_ROWS:
        rs = np.random.default_rng(D)
        C = 3
        tgt, otgt = big_problem(target, D, rs)
        q = tf(start(target, otgt, C, D, rs))
        imm = tf(np.ones(D, F))
        keys = tk(oprng.split(oprng.key(1), C))
        st = bj.hmc.init(q.clone(), tgt)
        eng = _engine.get_engine(st.position, tgt)
        eng.set_metric(imm)
        p = eng.sample_momentum(keys)
        ops = {
            "init": lambda: eng.init_state(q),
            "momentum": lambda: eng.sample_momentum(keys),
            "energy": lambda: eng.energy(p, st.logdensity),
            "leapfrog": lambda: eng.leapfrog_(q.clone(), p.clone(), st.logdensity.clone(), st.logdensity_grad.clone(),
                                              1e-3, 2),
            "hmc": lambda: bj.hmc.build_kernel()(keys, st, tgt, 1e-3, imm, 2),
            "mala": lambda: bj.mala.build_kernel()(keys, st, tgt, 1e-4),
            "barker": lambda: bj.barker.build_kernel()(keys, st, tgt, 1e-4, imm),
        }
        for op, fn in ops.items():
            got = _launched(fn)
            want = kernel_for(target, D, op)
            assert got == [want], f"{target} D={D} {op}: launched {got}, the table says {want}"
            seen.setdefault(want, set()).add((target, D))
    for name in sorted(seen):
        print(f"{name:28s} {sorted(seen[name])}")
    assert set(seen) == set().union(*(instances(t) for t in TARGETS))


# ---------------------------------------------------------------------------------------------------------------------
# building blocks
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("target, D, C, metric", BLOCK_CASES)
def test_building_blocks_match_oracle(target, D, C, metric):
    rs = np.random.default_rng(D + C)
    tgt, otgt = big_problem(target, D, rs)
    imm, om = make_metric(metric, C, D, rs)
    eng = engine(tgt, C, D, imm)
    q = start(target, otgt, C, D, rs)
    logp, g = eng.init_state(tf(q))
    lp0, g0 = otgt(q)
    close(npy(logp), lp0, scale=np.max(np.abs(lp0)) + D)
    close_row(npy(g), g0, target, D)
    keys = oprng.split(oprng.key(D), C)
    p0 = om.sample_momentum(keys, D)
    close(npy(eng.sample_momentum(tk(keys))), p0, rtol=3e-6)
    close(npy(eng.energy(tf(p0), logp)), -lp0 + om.kinetic_energy(p0), scale=np.max(np.abs(lp0)) + D)
    base = F(0.5 * step_size(target, D))
    for pce in (False, True):
        eps = (base * np.exp(rs.uniform(-0.5, 0.5, C))).astype(F) if pce else base
        for n in (0, 1, 5):
            dq, dp, dl, dg = tf(q), tf(p0), logp.clone(), g.clone()
            eng.leapfrog_(dq, dp, dl, dg, tf(eps) if pce else float(eps), n)
            if n == 0:   # nothing moves, bit for bit
                assert torch.equal(dq, tf(q)) and torch.equal(dp, tf(p0)) and torch.equal(dl, logp) and torch.equal(dg, g)
                continue
            q1, p1, lp1, g1 = ohmc.static_integration(otgt, om, q, p0, lp0, g0, eps[:, None] if pce else eps, n)
            rtol = 1e-5 if n == 1 else 2e-5
            close(npy(dq), q1, rtol=rtol)
            close_row(npy(dp), p1, target, D, rtol=rtol, neck_scale=max(1.0, float(np.max(eps)) * n * D))
            close_row(npy(dg), g1, target, D, rtol=rtol)
            close(npy(dl), lp1, scale=np.max(np.abs(lp1)) + D)
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# one HMC transition
# ---------------------------------------------------------------------------------------------------------------------
def hmc_step(tgt, q, keys, eps, imm, L, inplace):
    """One transition through bj.hmc with every info field; returns (new state, info, input state before the step)."""
    st = bj.hmc.init(tf(q), tgt)
    before = tuple(t.clone() for t in st)
    new, info = bj.hmc.build_kernel(full_info=True, inplace=inplace)(tk(keys), st, tgt, eps, tf(imm), L)
    torch.cuda.synchronize()
    return new, info, before


def compare_transition(target, D, keys, q, eps, om, onew, oinfo, new, info, before, lp0):
    """The fields of one transition against the oracle's; returns (device decisions, chains that agree)."""
    C = q.shape[0]
    e1, e1o = npy(info.energy), oinfo.energy
    e0o = (-lp0 + om.kinetic_energy(oinfo.momentum)).astype(F)
    delta_o = ohmc.safe_energy_diff(e0o, e1o)
    ok = np.isfinite(e1o) & ~oinfo.is_divergent   # a divergent trajectory: its flag, decision and carry-over only
    # the decision compares log u with min(delta, 0); an error de in either energy moves delta by de
    with np.errstate(invalid="ignore"):
        de = np.where(ok, np.abs(e1 - e1o), 0) + np.abs(npy(before[1]) - lp0) + 1e-6 * (np.abs(e0o) + D)
    close(npy(info.momentum), oinfo.momentum, rtol=3e-6)
    L = oinfo.num_integration_steps
    rtol = 1e-5 if L <= 1 else 2e-5
    close(npy(info.proposal.position)[ok], oinfo.proposal[0][ok], rtol=rtol)
    close_row(npy(info.proposal.momentum)[ok], oinfo.proposal[1][ok], target, D, rtol=rtol,
              neck_scale=max(1.0, float(np.max(eps)) * L * D))
    close(e1[ok], e1o[ok], scale=np.max(np.abs(e1o[ok]), initial=0) + D)
    assert (de[ok] <= 2e-5 * (np.abs(e0o[ok]) + D)).all(), np.max(de[ok])   # both energies within DESIGN's 1e-5
    u = oprng.uniform(oprng.split(keys, 2)[:, 1])
    with np.errstate(divide="ignore"):
        near = np.abs(np.log(u) - np.minimum(delta_o, 0)) <= 2 * de
        pa_tol = 1e-5 + 2 * de * oinfo.acceptance_rate
    pa = npy(info.acceptance_rate)
    assert (np.abs(pa - oinfo.acceptance_rate) <= pa_tol).all(), np.max(np.abs(pa - oinfo.acceptance_rate) / pa_tol)
    div = npy(info.is_divergent).astype(bool)
    assert ((div == oinfo.is_divergent) | (np.abs(-delta_o - 1000.0) <= 2 * de)).all()
    acc = npy(info.is_accepted).astype(bool)
    assert ((acc == oinfo.is_accepted) | near).all()
    same = acc == oinfo.is_accepted
    a = same & acc
    close(npy(new.position)[a], onew.position[a], rtol=rtol)
    close_row(npy(new.logdensity_grad)[a], onew.logdensity_grad[a], target, D, rtol=rtol)
    close(npy(new.logdensity)[a], onew.logdensity[a], scale=np.max(np.abs(onew.logdensity), initial=0) + D)
    # a rejected chain carries its input over bit for bit, in place or out of place
    r = torch.from_numpy(~acc).to(DEV)
    for got, was in zip(new, before):
        assert torch.equal(got[r], was[r])
    return acc, same


@pytest.mark.parametrize("target, D, C, metric, pce, inplace", HMC_CASES)
def test_hmc_transition_matches_oracle(target, D, C, metric, pce, inplace):
    rs = np.random.default_rng(3 * D + C)
    tgt, otgt = big_problem(target, D, rs)
    imm, om = make_metric(metric, C, D, rs)
    q = start(target, otgt, C, D, rs)
    lp0, g0 = otgt(q)
    base = F(step_size(target, D))
    eps = (base * np.exp(rs.uniform(-0.4, 0.4, C))).astype(F) if pce else base
    n_acc = 0
    for L in (0, 1, 6):
        keys = oprng.split(oprng.key(D + L), C)
        onew, oinfo = ohmc.hmc_kernel(keys, ohmc.HMCState(q, lp0, g0), otgt, eps, om, L)
        new, info, before = hmc_step(tgt, q, keys, tf(eps) if pce else float(eps), imm, L, inplace)
        acc, _ = compare_transition(target, D, keys, q, eps, om, onew, oinfo, new, info, before, lp0)
        if L == 0:   # no trajectory: the energy difference is exactly 0 and every chain moves to its own position
            assert acc.all() and torch.equal(new.position, before[0])
        n_acc += acc.sum()
    assert n_acc > 0
    if target in ("diag", "funnel", "hier"):   # NUTS is not built for these rows (the routing test pins the rest)
        with pytest.raises(bj.BjxError, match="dim <= 1024"):
            bj.nuts.build_kernel()(tk(keys), bj.hmc.init(tf(q), tgt), tgt, 0.01, tf(imm), 3)


@pytest.mark.parametrize("target, D, inplace", [("diag", 10756, True), ("funnel", 18432, False), ("hier", 10240, True),
                                                ("hier", 10244, False), ("user_diag", 18432, True)])
def test_unstable_step_sizes_diverge_and_reject(target, D, inplace):
    """Per-chain step sizes from stable to far past the stability limit: the unstable chains reach huge, infinite or NaN
    energies, and are flagged divergent and rejected with their state carried over bit for bit (in place: left alone), as
    the oracle decides.  Every k_big_hmc target class and k_big2 rejects here in one of the two output modes."""
    C = 9
    rs = np.random.default_rng(D + 1)
    tgt, otgt = big_problem(target, D, rs)
    imm, om = make_metric("diag", C, D, rs)
    q = start(target, otgt, C, D, rs)
    lp0, g0 = otgt(q)
    eps = (step_size(target, D) * np.array([0.5, 1, 3, 10, 30, 100, 1e3, 1e5, 1e7])).astype(F)
    keys = oprng.split(oprng.key(D), C)
    with np.errstate(all="ignore"):
        onew, oinfo = ohmc.hmc_kernel(keys, ohmc.HMCState(q, lp0, g0), otgt, eps, om, 6)
    new, info, before = hmc_step(tgt, q, keys, tf(eps), imm, 6, inplace)
    with np.errstate(all="ignore"):
        acc, _ = compare_transition(target, D, keys, q, eps, om, onew, oinfo, new, info, before, lp0)
    div = npy(info.is_divergent).astype(bool)
    assert div.sum() >= 3 and not div[0] and (~np.isfinite(oinfo.energy)).any() and (~np.isfinite(npy(info.energy))).any()
    assert not acc[div].any()


# ---------------------------------------------------------------------------------------------------------------------
# the native loop
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("target, D, C, off", NATIVE_CASES)
def test_native_sampler_equals_stepwise(target, D, C, off):
    """bjx_hmc_sample (one shared step key per transition, chain c folding in chain_offset + c on the device) against
    the step-wise transitions: run_inference_algorithm's loop, or with an offset, per-chain keys split explicitly."""
    rs = np.random.default_rng(D + off)
    tgt, otgt = big_problem(target, D, rs)
    q = tf(start(target, otgt, C, D, rs))
    imm = tf(np.exp(rs.uniform(-0.3, 0.3, D)).astype(F))
    eps = tf((step_size(target, D) * np.exp(rs.uniform(-0.3, 0.3, C))).astype(F))
    L, T_, thin = 4, 6, 2
    key = bj.random.key(D + off, DEV)
    st0 = bj.hmc.init(q, tgt)
    fin, hist, acc = bj.sample_hmc_native(key, st0, tgt, eps, imm, L, T_, chain_offset=off)
    if off == 0:
        st, steps = bj.run_inference_algorithm(key, bj.hmc(tgt, eps, imm, L), T_, initial_state=st0,
                                               transform=lambda s, i: (s.position, i.acceptance_rate))
    else:
        kern, st, steps = bj.hmc.build_kernel(), st0, []
        for k in bj.random.split(key, T_):
            st, info = kern(bj.random.split(k, off + C)[off:], st, tgt, eps, imm, L)
            steps.append((st.position, info.acceptance_rate))
    assert torch.equal(fin.position, st.position) and torch.equal(fin.logdensity, st.logdensity)
    assert torch.equal(fin.logdensity_grad, st.logdensity_grad)
    assert torch.equal(hist, torch.stack([s[0] for s in steps]))
    assert torch.equal(acc, torch.stack([s[1] for s in steps]))
    _, hist2, _ = bj.sample_hmc_native(key, st0, tgt, eps, imm, L, T_, thin=thin, chain_offset=off)
    assert torch.equal(hist2, hist[thin - 1::thin])
    assert float(acc.mean()) > 0
