"""Restatement of the rank-normalised diagnostics blackjax.rhat, ess_bulk and ess_tail (blackjax/diagnostics.py:92-155,
341-522; Vehtari et al. 2021) over a history [T, C, D], with the project's stated float64 positions and quantiles.
R-hat and ESS are oracle.diagnostics'.  TEST INFRASTRUCTURE."""
import numpy as np
from scipy.special import ndtri

from . import diagnostics as odiag

F = np.float32


def split_chains(x):
    """_split_chains (:357-364) of x [T, C, D] in the reference's chain-major axes: [2C, h, D], chain C + c holding the
    second half of chain c; an odd last draw is dropped."""
    x = np.asarray(x)
    h = x.shape[0] // 2
    xc = np.moveaxis(x[: 2 * h], 1, 0)                    # [C, 2h, D]
    return np.concatenate([xc[:, :h], xc[:, h:]], axis=0)


def pooled(x):
    """The n = 2C * h pooled draws per dimension in the order of x_split.reshape(n, D): index j = k * h + s."""
    xs = split_chains(x)
    return xs.reshape(xs.shape[0] * xs.shape[1], *xs.shape[2:])


def order(col):
    """Stable ascending order of a float32 column: -0 == +0, every NaN after +inf, ties by index."""
    return np.argsort(np.asarray(col, F), kind="stable")


def ranks(col):
    """1-based ranks of the stable order (argsort(argsort) + 1 of _rank_normalize, :396)."""
    o = order(col)
    r = np.empty(len(o), np.int64)
    r[o] = np.arange(1, len(o) + 1)
    return r


def blom(r, n):
    """Phi^-1((r - 3/8) / (n + 1/4)) with the position and Phi^-1 in float64, rounded to float32."""
    return ndtri((np.asarray(r, np.float64) - 0.375) / (float(n) + 0.25)).astype(F)


def lerp(a, b, t):
    """numpy's "linear" quantile between order statistics a <= b (float32) at fraction t, in float64."""
    if a == b:
        return float(a)
    a, b = float(a), float(b)
    diff = b - a
    return b - diff * (1.0 - t) if t >= 0.5 else a + diff * t


def quantile(col, q):
    """The pooled quantile at q: v = q (n - 1), the lerp of the order statistics floor(v), floor(v) + 1."""
    n = len(col)
    srt = np.asarray(col, F)[order(col)]
    v = q * (n - 1)
    i = int(np.floor(v))
    i = min(max(i, 0), n - 1)
    return lerp(srt[i], srt[min(i + 1, n - 1)], v - np.floor(v))


def median(col):
    """(a + b) * 0.5 in float32 over the order statistics floor((n - 1) / 2) and ceil((n - 1) / 2)."""
    n = len(col)
    srt = np.asarray(col, F)[order(col)]
    return (srt[(n - 1) // 2] + srt[n // 2]) * F(0.5)


def _scores_split(xs, folded):
    """Blom scores of the split draws xs [2C, h, D] (chain-major), optionally of |x - median| per dimension."""
    K, h = xs.shape[:2]
    flat = xs.reshape(K * h, -1)
    out = np.empty(flat.shape, F)
    for d in range(flat.shape[1]):
        col = flat[:, d]
        if folded:
            col = np.abs(col - median(col)).astype(F)
        out[:, d] = blom(ranks(col), len(col))
    return out.reshape(xs.shape)


def rank_normalize(x, folded=False):
    """The device layout of bjx_rank_normalize: [h, 2C, D] scores of the history x [T, C, D]."""
    return np.ascontiguousarray(np.moveaxis(_scores_split(split_chains(np.asarray(x, F)), folded), 0, 1))


def _nan_columns(x):
    return np.any(np.isnan(pooled(np.asarray(x, F))), axis=0)


def rhat(x):
    xs = split_chains(np.asarray(x, F))
    bulk = np.atleast_1d(odiag.potential_scale_reduction(_scores_split(xs, False), chain_axis=0, sample_axis=1))
    tail = np.atleast_1d(odiag.potential_scale_reduction(_scores_split(xs, True), chain_axis=0, sample_axis=1))
    out = np.maximum(bulk, tail)
    out[_nan_columns(x)] = np.nan
    return out


def ess_bulk(x):
    xs = split_chains(np.asarray(x, F))
    out = np.atleast_1d(odiag.effective_sample_size(_scores_split(xs, False), chain_axis=0, sample_axis=1)).astype(float)
    out[_nan_columns(x)] = np.nan
    return out


def indicators(x, prob=0.90):
    """(1[x <= q_lo], 1[x >= q_hi]) over the split draws [2C, h, D], the quantiles at (1 -+ prob) / 2, compared in float64."""
    xs = split_chains(np.asarray(x, F))
    flat = xs.reshape(xs.shape[0] * xs.shape[1], -1)
    q_lo = np.array([quantile(flat[:, d], (1.0 - prob) / 2.0) for d in range(flat.shape[1])])
    q_hi = np.array([quantile(flat[:, d], (1.0 + prob) / 2.0) for d in range(flat.shape[1])])
    x64 = xs.astype(np.float64)
    return (x64 <= q_lo).astype(np.float64), (x64 >= q_hi).astype(np.float64)


def ess_tail(x, prob=0.90):
    lo, hi = indicators(x, prob)
    e_lo = np.atleast_1d(odiag.effective_sample_size(lo, chain_axis=0, sample_axis=1))
    e_hi = np.atleast_1d(odiag.effective_sample_size(hi, chain_axis=0, sample_axis=1))
    out = np.minimum(e_lo, e_hi).astype(float)
    out[_nan_columns(x)] = np.nan
    return out
