"""The oracle of the rank-normalised diagnostics (oracle/rank_diagnostics.py) against independent restatements and the
reference's behavioural tests (tests/test_diagnostics.py, the rhat / ess_bulk / ess_tail classes; the ArviZ calibrations
are left out), and the sm_90a compile of bjx_rank.cu.  No GPU is needed."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
from scipy.stats import rankdata

from oracle import rank_diagnostics as ork

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
F = np.float32


@pytest.mark.parametrize("T", [4, 5, 10, 11])
def test_split_and_pooled_order(T):
    C, D = 3, 2
    x = np.arange(T * C * D, dtype=F).reshape(T, C, D)
    chains = np.moveaxis(x, 1, 0)                        # the reference's (nchains, nsamples, ...) axes
    h = T // 2
    expect = np.concatenate([chains[:, :h], chains[:, h:2 * h]], axis=0)
    np.testing.assert_array_equal(ork.split_chains(x), expect)
    np.testing.assert_array_equal(ork.pooled(x), expect.reshape(2 * C * h, D))
    # pooled index j = k * h + s: draw s of split chain k
    p = ork.pooled(x)
    for k in range(2 * C):
        for s in range(h):
            t, c = (s, k) if k < C else (h + s, k - C)
            np.testing.assert_array_equal(p[k * h + s], x[t, c])


def test_ranks_tie_free_match_rankdata():
    rs = np.random.default_rng(0)
    col = rs.standard_normal(1001).astype(F)
    np.testing.assert_array_equal(ork.ranks(col), rankdata(col, method="ordinal"))


def test_ranks_ties_zeros_and_nan_follow_stable_argsort():
    col = np.array([1.0, -0.0, 0.0, np.nan, np.inf, -np.inf, 1.0, 0.0, -0.0, np.nan, 1e-45, -1e-45], F)
    r = ork.ranks(col)
    np.testing.assert_array_equal(r, np.argsort(np.argsort(col, kind="stable"), kind="stable") + 1)
    # -0 and +0 are one value, ranked by index; NaNs come last, by index
    zeros = np.flatnonzero(col == 0)
    assert list(r[zeros]) == sorted(r[zeros]) and np.all(np.diff(r[zeros]) == 1)
    assert list(r[np.isnan(col)]) == [len(col) - 1, len(col)]
    assert r[4] == len(col) - 2                           # +inf just before the NaNs


def test_lerp_matches_numpy_linear_quantile():
    rs = np.random.default_rng(1)
    for n in (8, 20, 1000, 4097):
        col = rs.standard_normal(n).astype(F)
        for q in (0.05, 0.25, 0.5, 0.95, (1 - 0.9) / 2, (1 + 0.9) / 2):
            assert ork.quantile(col, q) == np.quantile(col.astype(np.float64), q, method="linear")


def test_blom_scores_in_float64():
    n = 40
    z = ork.blom(np.arange(1, n + 1), n)
    np.testing.assert_array_equal(z, np.array([__import__("statistics").NormalDist().inv_cdf((r - 0.375) / (n + 0.25))
                                               for r in range(1, n + 1)], np.float64).astype(F))
    assert np.all(np.diff(z) > 0) and abs(z[: n // 2].sum() + z[n // 2:].sum()) < 1e-5


def _draws(rs, C, T, D=1, shift=None, scale=None):
    x = rs.standard_normal((T, C, D)).astype(F)
    if shift is not None:
        x = x + np.asarray(shift, F)[None, :, None]
    if scale is not None:
        x = x * np.asarray(scale, F)[None, :, None]
    return x


def test_reference_rhat_recipes():
    rs = np.random.default_rng(2)
    assert abs(ork.rhat(_draws(rs, 4, 2000, 3)) - 1.0).max() < 0.01            # iid draws
    assert np.all(ork.rhat(_draws(rs, 4, 1000, 2, shift=[0, 0, 0, 3])) > 1.1)   # one chain shifted
    assert np.all(ork.rhat(_draws(rs, 4, 1000, 2, scale=[1, 1, 1, 4])) > 1.05)  # scale non-convergence (tail component)


def test_reference_ess_recipes():
    rs = np.random.default_rng(3)
    C, T = 4, 1000
    e = ork.ess_bulk(_draws(rs, C, T, 2))
    assert np.all((e > 0.5 * C * T) & (e < 2 * C * T))
    t = ork.ess_tail(_draws(rs, C, T, 2))
    assert np.all((t > 0.2 * C * T) & (t < 2 * C * T))
    ar = np.zeros((T, C, 2), F)                                                  # a poorly mixed chain: AR(1), phi = 0.95
    eps = rs.standard_normal((T, C, 2)).astype(F)
    for i in range(1, T):
        ar[i] = 0.95 * ar[i - 1] + eps[i]
    assert np.all(ork.ess_bulk(ar) < 0.5 * e) and np.all(ork.ess_tail(ar) < t)


def test_nan_columns_report_nan():
    rs = np.random.default_rng(4)
    x = _draws(rs, 3, 20, 3)
    x[5, 1, 1] = np.nan
    for f in (ork.rhat, ork.ess_bulk, ork.ess_tail):
        v = f(x)
        assert np.isnan(v[1]) and np.all(np.isfinite(v[[0, 2]]))


@pytest.mark.skipif(not os.path.exists(NVCC), reason="needs nvcc")
def test_rank_kernels_compile_without_spills(tmp_path):
    src = os.path.join(ROOT, "blackjax_b200", "csrc", "bjx_rank.cu")
    out = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                          "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "k.o")], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-2000:]
    blocks = [b for b in re.split(r"Compiling entry function", out.stderr) if "k_rank_" in b.split("\n")[0]]
    names = {re.search(r"k_rank_[a-z_]+", b.split("\n")[0]).group(0) for b in blocks}
    assert names == {"k_rank_keys", "k_rank_sort_tile", "k_rank_hist", "k_rank_scan", "k_rank_scatter", "k_rank_scores",
                     "k_rank_indicator", "k_rank_finish"}, names
    for b in blocks:
        assert " 0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in b, b
