"""MALA and Barker's proposal: the float32 oracles (oracle/mala.py, oracle/barker.py) against the reference's known
answers, the key tree, the NaN paths, the API surface and the ptxas report of the new kernels.  No GPU needed."""
import inspect
import re
import os
import shutil

import numpy as np
import pytest
from scipy import stats

from oracle import barker as ob
from oracle import mala as om
from oracle import prng
from oracle.targets import DiagGaussian, StdNormal

F = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def test_barker_nd_moments():
    """barker test_nd: 100k proposals from one state against the moments of the Barker pdf (trapezoid rule)."""
    n, D = 100_000, 2
    x = np.tile(np.array([0.5, -1.0], F), (n, 1))
    g = np.tile(np.array([1.0, -2.0], F), (n, 1))
    keys = prng.split(prng.key(0), n)
    y, _ = ob.sample(keys, x, g, F(0.5), ob.Metric(np.ones(D, F), n))  # (proposal, sign margins)
    grid = np.linspace(-6, 6, 20001)
    for i in range(D):
        t = grid * 0.5
        pdf = 2 * stats.norm.pdf(t, 0, 0.5) / (1 + np.exp(-g[0, i] * t))
        m1 = np.trapezoid(t * pdf, t)
        m2 = np.trapezoid(t * t * pdf, t)
        d = (y[:, i] - x[0, i]).astype(np.float64)
        assert abs(d.mean() - m1) < 5 * np.sqrt(m2 / n)
        assert abs((d * d).mean() - m2) < 0.02


def test_barker_preconditioning_matrix():
    """barker test_preconditioning_matrix: with the dense metric M^-1 = A the transitions are those of the identity
    metric on the target seen through q = M^1/2 u (M^1/2 = chol(A)^-T), same keys, positions mapped by M^1/2."""
    D, C = 3, 8
    A = np.array([[2.0, 0.3, 0.1], [0.3, 1.0, -0.2], [0.1, -0.2, 0.5]])
    Ms = np.linalg.inv(np.linalg.cholesky(A)).T
    prec = np.array([[1.5, 0.2, 0.0], [0.2, 0.8, 0.1], [0.0, 0.1, 1.2]])

    def logdensity(q):
        q = q.astype(np.float64)
        return (-0.5 * np.einsum("ci,ij,cj->c", q, prec, q)).astype(F), (-(q @ prec)).astype(F)

    def whitened(u):
        lp, gq = logdensity((u.astype(np.float64) @ Ms.T).astype(F))
        return lp, (gq.astype(np.float64) @ Ms).astype(F)

    u = np.random.default_rng(0).normal(size=(C, D)).astype(F)
    q = (u.astype(np.float64) @ Ms.T).astype(F)
    lq, gq = logdensity(q)
    lu, gu = whitened(u)
    key = prng.key(3)
    for t in range(10):
        keys = prng.split(prng.fold_in(key, t), C)
        (q, lq, gq), iq = ob.step(keys, q, lq, gq, logdensity, 0.7, A.astype(F))
        (u, lu, gu), iu = ob.step(keys, u, lu, gu, whitened, 0.7, None)
        np.testing.assert_allclose(q, u.astype(np.float64) @ Ms.T, rtol=2e-4, atol=2e-4)
        np.testing.assert_allclose(iq["acceptance_rate"], iu["acceptance_rate"], rtol=1e-3, atol=1e-4)


@pytest.mark.parametrize("eps, expect_high", [(1e-4, True), (50.0, False)])
def test_mala_acceptance_small_and_large_step(eps, expect_high):
    """mala test cases (tests/mcmc/test_mala.py:178-207): a tiny step accepts almost always, a huge one almost never."""
    C, D = 256, 5
    tgt = StdNormal(D)
    q = np.random.default_rng(1).normal(size=(C, D)).astype(F)
    lq, gq = tgt(q)
    _, info = om.step(prng.split(prng.key(7), C), q, lq, gq, tgt, eps)
    mean = info["acceptance_rate"].mean()
    assert (mean > 0.99) if expect_high else (mean < 0.01)


def test_key_tree():
    """MALA's noise is normal(split(key)[0]) and its accept uniform uses split(key)[1]; Barker's signs use
    split(split(split(key)[0])[1], 1)[0]."""
    key = prng.key(11)[None]
    q = np.zeros((1, 4), F)
    tgt = StdNormal(4)
    lq, gq = tgt(q)
    _, info = om.step(key, q, lq, gq, tgt, 0.1)
    xi = prng.normal(prng.split(key)[:, 0], (4,))
    np.testing.assert_allclose(info["proposal"][0], (np.sqrt(F(0.2)) * xi).astype(F), rtol=1e-6)
    u = prng.uniform(prng.split(key)[:, 1])
    assert info["margin"][0] == pytest.approx(abs(u[0] - info["acceptance_rate"][0]))
    np.testing.assert_array_equal(prng.split(prng.split(prng.split(key)[:, 0])[:, 1], 1)[:, 0], prng.fold_in(
        prng.fold_in(prng.fold_in(key, 0), 1), 0))


def test_nan_paths():
    """MALA maps a NaN log acceptance to -inf (p = 0); Barker keeps NaN: acceptance NaN and a rejection."""
    def nan_target(q):
        return np.full(q.shape[0], np.nan, F), np.full(q.shape, np.nan, F)

    q = np.zeros((2, 3), F)
    lq, gq = StdNormal(3)(q)
    keys = prng.split(prng.key(0), 2)
    (qm, _, _), im = om.step(keys, q, lq, gq, nan_target, 0.1)
    assert np.all(im["acceptance_rate"] == 0) and not im["is_accepted"].any()
    np.testing.assert_array_equal(qm, q)
    (qb, _, _), ib = ob.step(keys, q, lq, gq, nan_target, 0.1)
    assert np.all(np.isnan(ib["acceptance_rate"])) and not ib["is_accepted"].any()
    np.testing.assert_array_equal(qb, q)


def test_api_surface():
    import blackjax_b200 as bj
    from blackjax_b200.mcmc import barker, mala

    assert bj.barker_proposal is bj.barker
    assert list(inspect.signature(mala.as_top_level_api).parameters) == ["logdensity_fn", "step_size"]
    assert list(inspect.signature(barker.as_top_level_api).parameters) == ["logdensity_fn", "step_size",
                                                                           "inverse_mass_matrix"]
    assert mala.MALAState._fields == ("position", "logdensity", "logdensity_grad")
    assert mala.MALAInfo._fields == ("acceptance_rate", "is_accepted")
    assert barker.BarkerInfo._fields == ("acceptance_rate", "is_accepted", "proposal")
    assert callable(bj.sample_mala_native) and callable(bj.sample_barker_native)


# Every (row class, target, metric form) the library dispatches: each row class with the diagonal Gaussian and the funnel
# (diagonal metrics), the dense Gaussian and the banana at the row classes they run on, and Barker's small dense metric
# (DM) at every row class of at most 128 dims; the big rows with every built-in target.
ROWS = ["Row<1, false>", "Row<4, false>", "Row<4, true>", "Row<8, true>", "Row<16, true>", "Row<32, true>"]
SMALL = ["Row<1, false>", "Row<4, false>", "Row<4, true>"]
ROW_UNITS = {  # translation unit -> [(row, target, DM, kinds)]
    "diag": [(r, "TK_DIAG", "false", (0, 1)) for r in ROWS] + [(r, "TK_DIAG", "true", (1,)) for r in SMALL],
    "funnel": [(r, "TK_FUNNEL", "false", (0, 1)) for r in ROWS] + [(r, "TK_FUNNEL", "true", (1,)) for r in SMALL],
    "dense_banana": [(r, "TK_DENSE", "false", (0, 1)) for r in SMALL] + [(r, "TK_DENSE", "true", (1,)) for r in SMALL]
    + [("Row<1, false>", "TK_BANANA", dm, k) for dm, k in (("false", (0, 1)), ("true", (1,)))],
}
BIG_TARGETS = ["BJX_TARGET_DIAG_GAUSSIAN", "BJX_TARGET_FUNNEL", "BJX_TARGET_HIER_LOGIT"]
CLEAN = " 0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads"
# Known residuals, pinned so that they cannot grow (DESIGN §7): Barker's small dense-metric instances (DM = true, kind 1)
# keep a stack frame of at most 32 bytes around the noise draws' out-of-line square-root calls, and the hierarchical
# logit's CTA-row instances (target 4) spill at the 80-register cap of 768 threads (at most 88 bytes; k_big_hmc of that
# target keeps 32).
RESIDUAL = {r"k_langevin_(transition|chains)I.*ELb1ELi1EEEv": 32, r"k_big_langevinILi4E": 88}


def unit_source(name):
    lines = ['#include "bjx_big.cuh"', "namespace bjx {"]
    for row, tk, dm, kinds in ROW_UNITS.get(name, []):
        for kind in kinds:
            lines.append(f"template __global__ void k_langevin_transition<{row}, {tk}, {dm}, {kind}>(Params, const "
                         "uint32_t*, const float*, const float*, const float*, float*, float*, float*, LangevinArgs);")
            lines.append(f"template __global__ void k_langevin_chains<{row}, {tk}, {dm}, {kind}>(Params, float*, "
                         "float*, float*, LangevinArgs);")
    if name == "big":
        for tk in BIG_TARGETS:
            for kind in (0, 1):
                lines.append(f"template __global__ void k_big_langevin<{tk}, {kind}>(BigParams, const uint32_t*, "
                             "const float*, const float*, const float*, float*, float*, float*, LangevinArgs);")
    return "\n".join(lines + ["}"]) + "\n"


@pytest.mark.skipif(not os.path.exists(NVCC), reason="needs nvcc")
def test_kernels_compile_without_spills(tmp_path):
    """Every MALA / Barker kernel instance the library builds compiles with no stack frame and no spills (ptxas -v), the
    units compiled in parallel."""
    import subprocess
    units = list(ROW_UNITS) + ["big"]
    procs = {}
    for u in units:
        (tmp_path / f"{u}.cu").write_text(unit_source(u))
        procs[u] = subprocess.Popen([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas",
                                     "-v", "-I", os.path.join(ROOT, "blackjax_b200", "csrc"), "-I",
                                     os.path.join(ROOT, "include"), "-c", str(tmp_path / f"{u}.cu"), "-o",
                                     str(tmp_path / f"{u}.o")], stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                                    text=True)
    bad = []
    for u, p in procs.items():
        _, err = p.communicate()
        assert p.returncode == 0, err[-2000:]
        blocks = [b for b in err.split("Compiling entry function") if "langevin" in b.split("\n")[0]]
        expect = (2 * sum(len(k) for *_, k in ROW_UNITS[u])) if u != "big" else 2 * len(BIG_TARGETS)
        assert len(blocks) == expect, (u, len(blocks))
        for b in blocks:
            if CLEAN in b:
                continue
            name = b.split("\n")[0]
            frame = int(re.search(r"(\d+) bytes stack frame", b).group(1))
            bound = next((v for k, v in RESIDUAL.items() if re.search(k, name)), None)
            if bound is None or frame > bound:
                bad.append(" ".join(b.split("\n")[:2]))
    assert not bad, "\n".join(bad)
