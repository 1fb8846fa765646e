"""Slice sampling: the float32 oracle (oracle/slice_sampling.py) against the reference's known answers
(tests/mcmc/test_slice.py), explicit compositions of the key tree, _best_interval, the bisection cap, the API surface and
the ptxas report of the new kernels.  No GPU needed."""
import inspect
import os
import re
import shutil

import numpy as np
import pytest

from oracle import prng
from oracle import slice_sampling as osl
from oracle.targets import StdNormal

F = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
INTERVALS = ["doubling", "stepping_out"]


def run_chain(fn, x0, n, seed=0, **kw):
    """n transitions of one chain; returns positions [n, D] and is_accepted [n]."""
    x = np.asarray(x0, F)[None]
    lp = fn(x)[0]
    xs, acc = [], []
    for k in prng.split(prng.key(seed), n):
        (x, lp), info = osl.step(k[None], x, lp, fn, **kw)
        xs.append(x[0])
        acc.append(info["is_accepted"][0])
    return np.array(xs), np.array(acc)


@pytest.mark.parametrize("interval", INTERVALS)
def test_brackets_contain_origin_and_leave_slice(interval):
    """test_slice.py: the bracket of a standard normal from its mode holds t = 0 and has expanded (doubling: past
    |t| = 3)."""
    fn = StdNormal(1)
    (_, _), info = osl.step(prng.key(0)[None], np.zeros((1, 1), F), fn(np.zeros((1, 1), F))[0], fn, width=1.0,
                            interval=interval)
    assert info["bracket_left"][0] <= 0 <= info["bracket_right"][0]
    assert info["num_expansions"][0] > 0
    if interval == "doubling":
        assert info["bracket_left"][0] < -3 or info["bracket_right"][0] > 3
    else:
        assert info["bracket_right"][0] - info["bracket_left"][0] > 1.0


@pytest.mark.parametrize("scale", [1.0, 2.5, [0.5, 2.0, 1.0], [[1.0, 0.0, 0.0], [0.5, 2.0, 0.0], [0.1, 0.2, 0.5]]])
def test_direction_is_unit_norm(scale):
    d = osl.direction(prng.split(prng.key(1), 16), 3, np.asarray(scale, F))
    np.testing.assert_allclose(np.linalg.norm(d.astype(np.float64), axis=1), 1.0, atol=1e-6)


def test_vector_scale_tilts_direction():
    d = osl.direction(prng.split(prng.key(2), 500), 2, np.array([10.0, 0.1], F))
    m = np.abs(d).mean(axis=0)
    assert m[0] > m[1]


@pytest.mark.parametrize("interval", INTERVALS)
def test_step_shapes(interval):
    fn = StdNormal(3)
    C = 5
    x = np.zeros((C, 3), F)
    (xn, ln), info = osl.step(prng.split(prng.key(0), C), x, fn(x)[0], fn, interval=interval)
    assert xn.shape == (C, 3) and ln.shape == (C,)
    np.testing.assert_allclose(ln, fn(xn)[0], rtol=1e-6)
    for k in ("is_accepted", "num_expansions", "num_shrink", "bracket_left", "bracket_right", "margin"):
        assert info[k].shape == (C,)


@pytest.mark.parametrize("interval", INTERVALS)
def test_isotropic_std_normal_moments(interval):
    s, acc = run_chain(StdNormal(1), [0.0], 1500, seed=3, interval=interval)
    assert abs(s.mean()) < 0.12 and abs(s.std() - 1.0) < 0.12 and acc.all()


@pytest.mark.parametrize("interval", INTERVALS)
def test_correlated_gaussian_dense_scale(interval):
    sigma = np.array([[1.0, 0.8], [0.8, 1.0]])
    prec = np.linalg.inv(sigma)

    def fn(q):
        q = np.asarray(q, F)
        return (-0.5 * np.einsum("ni,ij,nj->n", q, prec, q)).astype(F), None

    s, _ = run_chain(fn, [0.0, 0.0], 1500, seed=4, scale=np.linalg.cholesky(sigma).astype(F), interval=interval)
    np.testing.assert_allclose(np.cov(s[200:].T), sigma, atol=0.3)


def test_nonzero_mean():
    def fn(q):
        q = np.asarray(q, F)
        return (-0.5 * np.sum((q - 3.0) ** 2, axis=1)).astype(F), None

    s, _ = run_chain(fn, [0.0], 1500, seed=5)
    assert abs(s[200:].mean() - 3.0) < 0.15


@pytest.mark.parametrize("interval", INTERVALS)
def test_skewed_exponential(interval):
    """Exp(1) per axis (-inf outside the positive orthant): mean 1, sd 1, right-skewed, never outside."""
    def fn(q):
        q = np.asarray(q, F)
        return np.where(np.all(q > 0, axis=1), -np.sum(q, axis=1), -np.inf).astype(F), None

    s, acc = run_chain(fn, [1.0, 1.0], 1500, seed=6, interval=interval)
    assert (s > 0).all() and acc.mean() > 0.99
    np.testing.assert_allclose(s.mean(axis=0), 1.0, atol=0.25)
    skew = np.mean(((s - s.mean(0)) / s.std(0)) ** 3, axis=0)
    assert (skew > 1.0).all()


def test_best_interval():
    assert osl.best_interval([0, 0, 1, 0, 1]) == 2
    assert osl.best_interval([1, 1, 1]) == 0
    assert osl.best_interval([0, 0, 0, 0]) == 3


@pytest.mark.parametrize("interval", INTERVALS)
def test_key_tree_composed_explicitly(interval):
    """The direction, the level, the interval's draws and the shrink key chain, composed from oracle.prng."""
    D, width, me = 4, F(0.7), 10
    key = prng.key(9)
    x = np.full((1, D), 0.3, F)
    fn = StdNormal(D)
    lp = fn(x)[0]
    (_, _), info = osl.step(key[None], x, lp, fn, width=width, interval=interval, max_expansions=me, max_shrinkage=1)
    prop_key, slice_key = prng.fold_in(key, 0), prng.fold_in(key, 1)
    z = prng.normal(prop_key, (D,))
    np.testing.assert_array_equal(info["direction"][0], (z / F(np.sqrt(np.sum(z.astype(np.float64) ** 2)))).astype(F))
    interval_key, shrink_key = prng.fold_in(slice_key, 1), prng.fold_in(slice_key, 2)
    if interval == "doubling":
        l0 = F(-width * prng.uniform(prng.fold_in(interval_key, 0)))
        side = prng.uniform(prng.fold_in(interval_key, 1), (me + 1,)) < F(0.5)
        j = info["num_expansions"][0]
        inc_l = sum(float(width) * 2.0 ** i for i in range(j) if side[i])
        inc_r = sum(float(width) * 2.0 ** i for i in range(j) if not side[i])
        assert info["bracket_left"][0] == F(l0 - F(inc_l))
        assert info["bracket_right"][0] == F(F(l0 + width) + F(inc_r))
    else:
        left = F(-width * prng.uniform(prng.fold_in(interval_key, 0)))
        j = int(np.floor(F(F(me) * prng.uniform(prng.fold_in(interval_key, 1)))))
        k = me - 1 - j
        n_l = round(float(left - info["bracket_left"][0]) / float(width))
        n_r = round(float(info["bracket_right"][0] - F(left + width)) / float(width))
        assert 0 <= n_l <= j and 0 <= n_r <= max(k, 0) and info["num_expansions"][0] == n_l + n_r
    # the first shrinkage try: t = left + uniform(split(shrink_key)[1]) (right - left)
    sub = prng.fold_in(shrink_key, 1)
    t = F(info["bracket_left"][0] + F(prng.uniform(sub) * F(info["bracket_right"][0] - info["bracket_left"][0])))
    assert info["num_shrink"][0] == 1
    lvl = F(lp[0] + np.log(prng.uniform(prng.fold_in(slice_key, 0))))
    pt = (x[0] + (t * info["direction"][0]).astype(F)).astype(F)
    if not info["is_accepted"][0]:
        assert fn(pt[None])[0][0] < lvl or interval == "doubling"


def test_bisection_cap_binds_only_on_overflow():
    """A finite doubling bracket reaches 1.1 width within max_expansions passes; a bracket whose width overflowed keeps
    an infinite mid, which the cap alone stops."""
    def always_in(t):
        return True

    me = 10
    width = F(1.0)
    right = F(width * 2 ** me - 0.25)
    ok, passes = osl.doubling_accept(always_in, F(0.1), F(-0.25), right, width, me + 1)
    assert ok and passes <= me
    ok, passes = osl.doubling_accept(always_in, F(0.1), F(-np.inf), F(np.inf), width, me + 1)
    assert passes == me + 1


def test_caps_zero():
    """max_shrinkage = 0 keeps the state and reports no acceptance; max_expansions = 0 keeps the initial bracket."""
    fn = StdNormal(2)
    x = np.full((3, 2), 0.5, F)
    keys = prng.split(prng.key(4), 3)
    (xn, ln), info = osl.step(keys, x, fn(x)[0], fn, max_shrinkage=0)
    np.testing.assert_array_equal(xn, x)
    assert not info["is_accepted"].any() and (info["num_shrink"] == 0).all()
    (_, _), info = osl.step(keys, x, fn(x)[0], fn, max_expansions=0)
    np.testing.assert_allclose(info["bracket_right"] - info["bracket_left"], 1.0, rtol=1e-6)
    assert (info["num_expansions"] == 0).all()


def test_api_surface():
    import blackjax_b200 as bj
    from blackjax_b200.mcmc import slice as sl
    assert bj.slice_sampling is not None and callable(bj.sample_slice_sampling_native)
    assert sl.SliceState._fields == ("position", "logdensity")
    assert sl.SliceInfo._fields == ("is_accepted", "num_expansions", "num_shrink", "bracket_left", "bracket_right")
    sig = inspect.signature(sl.as_top_level_api)
    assert list(sig.parameters) == ["logdensity_fn", "proposal_generator", "width", "interval", "max_expansions",
                                    "max_shrinkage"]
    assert sig.parameters["width"].default == 1.0 and sig.parameters["interval"].default is sl.doubling
    assert sig.parameters["max_expansions"].default == 10 and sig.parameters["max_shrinkage"].default == 100
    assert list(inspect.signature(sl.build_kernel).parameters)[:3] == ["interval", "max_expansions", "max_shrinkage"]
    with pytest.raises(NotImplementedError, match="doubling and stepping_out"):
        sl.build_kernel(interval=lambda *a: None)
    with pytest.raises(NotImplementedError, match="direction_proposal"):
        sl.as_top_level_api(lambda x: x, proposal_generator=lambda k, p, f: None)
    with pytest.raises(ValueError, match=">= 0"):
        sl.build_kernel(max_shrinkage=-1)


ROWS = ["Row<1, false>", "Row<4, false>", "Row<4, true>", "Row<8, true>", "Row<16, true>", "Row<32, true>"]
SMALL = ["Row<1, false>", "Row<4, false>", "Row<4, true>"]
# translation unit -> [(row, target, DM)]: both kernels of each
ROW_UNITS = {
    "diag": [(r, "TK_DIAG", "false") for r in ROWS] + [(r, "TK_DIAG", "true") for r in SMALL],
    "funnel": [(r, "TK_FUNNEL", "false") for r in ROWS] + [(r, "TK_FUNNEL", "true") for r in SMALL],
    "dense_banana": [(r, "TK_DENSE", dm) for r in SMALL for dm in ("false", "true")]
    + [("Row<1, false>", "TK_BANANA", dm) for dm in ("false", "true")],
}
BIG_TARGETS = ["BJX_TARGET_DIAG_GAUSSIAN", "BJX_TARGET_FUNNEL", "BJX_TARGET_HIER_LOGIT"]
CLEAN = " 0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads"
# Known residuals, pinned so that they cannot grow (DESIGN §7): the slice machine's state stays live across the target's
# evaluation, and some instances keep a small stack frame for it; the hierarchical logit on the CTA rows, whose 768
# threads have 80 registers each, keeps a larger one.  Every other instance is clean.
RESIDUAL = {r"k_slice_(transition|chains)INS_3RowILi\d+ELb\dEEELi\dELb\dEEEv": 56, r"k_big_sliceILi4EEEv": 500}


def unit_source(name):
    lines = ['#include "bjx_big.cuh"', "namespace bjx {"]
    for row, tk, dm in ROW_UNITS.get(name, []):
        lines.append(f"template __global__ void k_slice_transition<{row}, {tk}, {dm}>(Params, const uint32_t*, "
                     "const float*, const float*, float*, float*, SliceArgs);")
        lines.append(f"template __global__ void k_slice_chains<{row}, {tk}, {dm}>(Params, float*, float*, SliceArgs);")
    if name == "big":
        for tk in BIG_TARGETS:
            lines.append(f"template __global__ void k_big_slice<{tk}>(BigParams, const uint32_t*, const float*, "
                         "const float*, float*, float*, SliceArgs);")
    return "\n".join(lines + ["}"]) + "\n"


@pytest.mark.skipif(not os.path.exists(NVCC), reason="needs nvcc")
def test_kernels_compile_without_spills(tmp_path):
    """Every slice sampling kernel instance the library builds compiles with no stack frame and no spills (ptxas -v),
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
        blocks = [b for b in err.split("Compiling entry function") if "_slice" in b.split("\n")[0]]
        expect = 2 * len(ROW_UNITS[u]) if u != "big" else len(BIG_TARGETS)
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
