"""Elliptical slice sampling: the float32 oracle (oracle/elliptical_slice.py) against the reference's known answers
(tests/mcmc/test_elliptical_slice.py), the key tree, NaN proposals, the sub-iteration cap, the API surface and the ptxas
report of the new kernels.  No GPU needed."""
import inspect
import os
import re
import shutil

import numpy as np
import pytest

from oracle import elliptical_slice as oe
from oracle import prng
from oracle.targets import DiagGaussian

F = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def flat(q):
    return np.zeros(q.shape[0], F), np.zeros_like(q)


def test_ellipse_known_points():
    """test_elliptical_slice.py: theta = 0 returns (x, nu), theta = pi negates both about the mean, theta = pi / 2
    swaps them, and the squared norm about the mean is preserved."""
    rs = np.random.default_rng(0)
    x, nu = rs.normal(size=(2, 1, 5)).astype(F)
    mean = rs.normal(size=5).astype(F)
    for theta, ep, em in ((0.0, x, nu), (np.pi, 2 * mean - x, 2 * mean - nu), (np.pi / 2, nu, 2 * mean - x)):
        t = np.array([theta], F)
        p = oe.ellipse(x, nu, mean, t)
        m = oe.ellipse(nu, x, mean, -t)  # (nu - mu) cos t - (x - mu) sin t + mu, as sin(-t) = -sin(t)
        np.testing.assert_allclose(p, ep, atol=1e-5)
        np.testing.assert_allclose(m, em, atol=1e-5)
        n0 = np.sum((x - mean) ** 2) + np.sum((nu - mean) ** 2)
        n1 = np.sum((p - mean) ** 2) + np.sum((m - mean) ** 2)
        np.testing.assert_allclose(n1, n0, rtol=1e-5)


def test_step_invariants():
    """subiter >= 1, the stored log-likelihood is the likelihood at the new position, and the info's momentum pairs
    with the position on the same ellipse (norm preserved); a flat likelihood always accepts the first proposal."""
    C, D = 64, 6
    rs = np.random.default_rng(1)
    lik = DiagGaussian(0.7, D)
    x = rs.normal(size=(C, D)).astype(F)
    keys = prng.split(prng.key(2), C)
    mean = np.full(D, 0.3, F)
    scale = oe.prior_scale(np.full(D, 2.0, F))
    (xn, ln), info = oe.step(keys, x, lik(x)[0], lik, mean, scale)
    assert np.all(info["subiter"] >= 1) and not info["exhausted"].any()
    np.testing.assert_array_equal(ln, lik(xn)[0])
    n0 = np.sum((x - mean) ** 2 + (info["nu"] - mean) ** 2, axis=1)
    n1 = np.sum((xn - mean) ** 2 + (info["momentum"] - mean) ** 2, axis=1)
    np.testing.assert_allclose(n1, n0, rtol=1e-4)
    (xf, lf), fi = oe.step(keys, x, np.zeros(C, F), flat, mean, scale)
    assert np.all(fi["subiter"] == 1) and np.all(np.isfinite(xf)) and np.all(lf == 0)


def test_wrong_cov_dims():
    with pytest.raises(ValueError, match="wrong number of dimensions"):
        oe.prior_scale(np.ones((2, 2, 2), F))


def test_key_tree():
    """The 4-way split, fold_in(key_slice, 1) as the first redraw and the float32 2 pi, composed explicitly."""
    C, D = 16, 3
    keys = prng.split(prng.key(7), C)
    x = np.random.default_rng(3).normal(size=(C, D)).astype(F)
    mean = np.zeros(D, F)
    scale = oe.prior_scale(np.ones(D, F))
    # a likelihood that rejects every first proposal (logL(x) = 0 above the slice, -1e30 elsewhere) until the bracket
    # brings the proposal back within 1e-3 of x
    x0 = x.copy()

    def near(q):
        d = np.max(np.abs(q - x0), axis=1)
        return np.where(d < 1e-3, F(0), F(-1e30)).astype(F), np.zeros_like(q)

    (_, _), info = oe.step(keys, x, np.zeros(C, F), near, mean, scale, max_subiter=2)
    ks = np.stack([prng.fold_in(keys, i) for i in range(4)], axis=1)
    np.testing.assert_array_equal(prng.split(keys, 4), ks)
    z = prng.normal(ks[:, 1], (D,))
    np.testing.assert_array_equal(info["nu"], z)
    theta0 = (F(6.2831855) * prng.uniform(ks[:, 3])).astype(F)
    assert F(2 * np.pi) == F(6.2831855)
    f = prng.uniform(prng.fold_in(ks[:, 0], 1))
    lo, hi = (theta0 - F(6.2831855)).astype(F), theta0
    theta1 = np.maximum(lo, (f * (hi - lo)).astype(F) + lo).astype(F)
    moved = ~info["exhausted"]
    np.testing.assert_array_equal(info["theta"][moved], theta1[moved])
    assert np.all(info["subiter"] == 2)
    assert np.all(info["theta"][info["exhausted"]] == 0)


def test_nan_proposal_accepted():
    """jax.lax.while_loop(logL(p) <= logy) ends on a NaN: the NaN proposal is the new state."""
    C, D = 8, 4
    keys = prng.split(prng.key(11), C)
    x = np.ones((C, D), F)

    def nan_lik(q):
        return np.full(q.shape[0], np.nan, F), np.zeros_like(q)

    (xn, ln), info = oe.step(keys, x, np.zeros(C, F), nan_lik, np.zeros(D, F), oe.prior_scale(np.ones(D, F)))
    assert np.all(np.isnan(ln)) and np.all(info["subiter"] == 1) and not info["exhausted"].any()
    assert not np.array_equal(xn, x)


def test_cap_keeps_state():
    """A start at logL = -inf never leaves the loop in the reference; with the cap the chain keeps (x, logL(x)) and
    reports exhausted, subiter = max_subiter, theta = 0 and momentum = nu."""
    C, D = 8, 5
    keys = prng.split(prng.key(5), C)
    x = np.random.default_rng(4).normal(size=(C, D)).astype(F)

    def ninf(q):
        return np.full(q.shape[0], -np.inf, F), np.zeros_like(q)

    (xn, ln), info = oe.step(keys, x, np.full(C, -np.inf, F), ninf, np.zeros(D, F), oe.prior_scale(np.ones(D, F)),
                             max_subiter=37)
    assert info["exhausted"].all() and np.all(info["subiter"] == 37) and np.all(info["theta"] == 0)
    np.testing.assert_array_equal(xn, x)
    assert np.all(ln == -np.inf)
    np.testing.assert_array_equal(info["momentum"], info["nu"])


def test_api_surface():
    """blackjax.elliptical_slice: the reference's names, signatures and defaults, plus max_subiter and exhausted."""
    import blackjax_b200 as bj
    from blackjax_b200.mcmc import elliptical_slice as es
    assert bj.elliptical_slice is not None
    assert es.EllipSliceState._fields == ("position", "logdensity")
    assert es.EllipSliceInfo._fields == ("momentum", "theta", "subiter", "exhausted")
    sig = inspect.signature(es.as_top_level_api)
    assert list(sig.parameters) == ["loglikelihood_fn", "mean", "cov", "max_subiter"]
    assert sig.parameters["max_subiter"].default == 1000
    assert list(inspect.signature(es.build_kernel).parameters)[:3] == ["cov_matrix", "mean", "max_subiter"]
    with pytest.raises(ValueError, match="wrong number of dimensions"):
        es.build_kernel(np.ones((2, 2, 2), F), 0.0)
    assert callable(bj.sample_elliptical_slice_native)


ROWS = ["Row<1, false>", "Row<4, false>", "Row<4, true>", "Row<8, true>", "Row<16, true>", "Row<32, true>"]
SMALL = ["Row<1, false>", "Row<4, false>", "Row<4, true>"]
TC = ["Row<8, true>", "Row<16, true>", "Row<32, true>"]
# translation unit -> [(row, target, DM, prior, with the native loop)]
ROW_UNITS = {
    "diag": [(r, "TK_DIAG", "false", 0, True) for r in ROWS] + [(r, "TK_DIAG", "false", 2, False) for r in TC]
    + [(r, "TK_DIAG", "true", 1, True) for r in SMALL],
    "funnel": [(r, "TK_FUNNEL", "false", 0, True) for r in ROWS] + [(r, "TK_FUNNEL", "false", 2, False) for r in TC]
    + [(r, "TK_FUNNEL", "true", 1, True) for r in SMALL],
    "dense_banana": [(r, "TK_DENSE", dm, p, True) for r in SMALL for dm, p in (("false", 0), ("true", 1))]
    + [("Row<1, false>", "TK_BANANA", dm, p, True) for dm, p in (("false", 0), ("true", 1))],
}
BIG_TARGETS = ["BJX_TARGET_DIAG_GAUSSIAN", "BJX_TARGET_FUNNEL", "BJX_TARGET_HIER_LOGIT"]
CLEAN = " 0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads"
# Known residuals, pinned so that they cannot grow (DESIGN §7): the dense Gaussian target's instances (target 2), whose
# precision matvec runs inside the slice loop, keep a stack frame of at most 20 bytes, and the funnel's native loop with a
# small dense prior (Row<4, true>, DM = true, prior 1) one of 8.  Every other instance is clean.
RESIDUAL = {r"k_ess_(transition|chains)INS_3RowILi\d+ELb\dEEELi2E": 20, r"k_ess_chainsINS_3RowILi4ELb1EEELi1ELb1ELi1E": 8}


def unit_source(name):
    lines = ['#include "bjx_big.cuh"', "namespace bjx {"]
    for row, tk, dm, prior, chains in ROW_UNITS.get(name, []):
        lines.append(f"template __global__ void k_ess_transition<{row}, {tk}, {dm}, {prior}>(Params, const uint32_t*, "
                     "const float*, const float*, float*, float*, EssArgs);")
        if chains:
            lines.append(f"template __global__ void k_ess_chains<{row}, {tk}, {dm}, {prior}>(Params, float*, float*, "
                         "EssArgs);")
    if name == "big":
        for tk in BIG_TARGETS:
            lines.append(f"template __global__ void k_big_ess<{tk}>(BigParams, const uint32_t*, const float*, "
                         "const float*, float*, float*, EssArgs);")
    return "\n".join(lines + ["}"]) + "\n"


@pytest.mark.skipif(not os.path.exists(NVCC), reason="needs nvcc")
def test_kernels_compile_without_spills(tmp_path):
    """Every elliptical slice kernel instance the library builds compiles with no stack frame and no spills (ptxas -v),
    the units compiled in parallel."""
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
        blocks = [b for b in err.split("Compiling entry function") if "_ess" in b.split("\n")[0]]
        expect = sum(1 + int(c) for *_, c in ROW_UNITS[u]) if u != "big" else len(BIG_TARGETS)
        assert len(blocks) == expect, (u, len(blocks))
        for b in blocks:
            if CLEAN in b:
                continue
            name = b.split("\n")[0]
            frame = int(re.search(r"(\d+) bytes stack frame", b).group(1))
            spill = max(int(v) for v in re.findall(r"(\d+) bytes spill", b))
            bound = next((v for k, v in RESIDUAL.items() if re.search(k, name)), None)
            if bound is None or max(frame, spill) > bound:
                bad.append(" ".join(b.split("\n")[:3]))
    assert not bad, "\n".join(bad)
