"""The rank-normalised diagnostics on the device (bjx_rank_normalize, bjx_rank_diagnostics; blackjax.rhat, ess_bulk,
ess_tail) against oracle/rank_diagnostics.py.

Bars: scores within 1 float32 ulp and, up to n = 2^22 pooled draws, in exactly the oracle's rank order (the tie-break);
R-hat within rtol 2e-5; ESS by the rule of the existing ESS test (90 % of columns within 2e-3, all within 0.2: Geyer's
truncation sits on float ties); NaN columns NaN in all three outputs."""
import numpy as np
import pytest
import torch

import blackjax_b200 as bj
from blackjax_b200 import _lib, targets as T
from blackjax_b200._engine import get_engine
from blackjax_b200._lib import BjxError, check, ptr
from oracle import rank_diagnostics as ork

pytestmark = pytest.mark.gpu
F = np.float32
DEV = "cuda:0"


def tf(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=F)).to(DEV)


def npy(t):
    return t.detach().cpu().numpy()


def ess_rule(ess, ref):
    np.testing.assert_array_equal(np.isnan(ess), np.isnan(ref))
    ok = ~np.isnan(ref)
    ess, ref = ess[ok], ref[ok]
    rel = np.abs(ess - ref) / np.maximum(np.abs(ref), 1e-30)
    rel[ref == 0] = np.abs(ess[ref == 0])
    assert np.mean(rel < 2e-3) >= 0.9, (ess, ref)
    assert np.all(rel < 0.2), (ess, ref)


def ar1(rs, T_, C, D):
    phi = np.linspace(-0.6, 0.95, D).astype(F)
    e = rs.standard_normal((T_, C, D)).astype(F)
    x = np.zeros((T_, C, D), F)
    x[0] = e[0]
    for t in range(1, T_):
        x[t] = phi * x[t - 1] + e[t]
    return x


def special(rs, T_, C, D):
    """AR(1) columns with a constant column, a two-valued one, mixed +-0 / +-inf / subnormals and heavy ties."""
    x = ar1(rs, T_, C, D)
    vals = np.array([0.0, -0.0, np.inf, -np.inf, 1e-45, -1e-45, 1e-40, 1.0, -1.0], F)
    for d in range(D):
        kind = d % 4
        if kind == 1:
            x[..., d] = 2.5
        elif kind == 2:
            x[..., d] = np.where(rs.random((T_, C)) < 0.3, F(1.0), F(-2.0))
        elif kind == 3:
            x[..., d] = vals[rs.integers(0, len(vals), (T_, C))]
    return x


def hmc_history(T_, C, D):
    """An HMC history at a step size with low acceptance: rejected transitions repeat draws exactly."""
    tgt = T.StdNormal(D)
    st0 = bj.hmc.init(torch.randn(C, D, device=DEV, generator=torch.Generator(DEV).manual_seed(1)), tgt)
    _, hist, acc = bj.sample_hmc_native(bj.random.key(11, DEV), st0, tgt, 1.95, torch.ones(D, device=DEV), 3, T_)
    h = npy(hist)
    assert np.mean(h[1:] == h[:-1]) > 0.1, "expected many rejected transitions"
    return h


def check_all(x, prob=0.9, exact_order=True):
    T_, C, D = x.shape
    tgt = T.StdNormal(D)
    hx = tf(x)
    for folded in (False, True):
        dev = npy(bj.diagnostics.rank_normalize(hx, tgt, folded=folded))
        ref = ork.rank_normalize(x, folded=folded)
        assert dev.shape == ref.shape == (T_ // 2, 2 * C, D)
        np.testing.assert_array_max_ulp(dev, ref, maxulp=1)
        if exact_order:
            dp, xp = np.moveaxis(dev, 0, 1).reshape(-1, D), ork.pooled(x)
            for d in range(D):
                col = xp[:, d] if not folded else np.abs(xp[:, d] - ork.median(xp[:, d])).astype(F)
                np.testing.assert_array_equal(np.argsort(dp[:, d], kind="stable"), ork.order(col))
    rh = npy(bj.rhat(hx, tgt))
    np.testing.assert_allclose(rh, ork.rhat(x), rtol=2e-5, equal_nan=True)
    ess_rule(npy(bj.ess_bulk(hx, tgt)), ork.ess_bulk(x))
    ess_rule(npy(bj.ess_tail(hx, tgt, prob=prob)), ork.ess_tail(x, prob))


# (T, C, D): T = 4, odd T, C = 1, D = 1, n = 2C * (T // 2) one below, at and one above the single-tile edge (4096), and
# several tiles
SHAPES = [(4, 1, 1), (5, 2, 3), (9, 3, 7), (4094, 1, 2), (4095, 1, 2), (256, 16, 3), (4098, 1, 2), (257, 8, 5),
          (1000, 64, 40), (63, 200, 33)]


@pytest.mark.parametrize("shape", SHAPES)
def test_ar1_against_oracle(shape):
    rs = np.random.default_rng(sum(shape))
    check_all(ar1(rs, *shape))


@pytest.mark.parametrize("shape", [(9, 3, 8), (4095, 1, 4), (300, 20, 8)])
def test_ties_zeros_infinities_subnormals(shape):
    rs = np.random.default_rng(7)
    check_all(special(rs, *shape))


def test_quantile_on_a_tie():
    """The lower 5 % quantile of a column of mostly one value sits on a tie: 1[x <= q_lo] counts the whole tie."""
    rs = np.random.default_rng(8)
    x = np.where(rs.random((400, 8, 2)) < 0.5, F(0.0), rs.standard_normal((400, 8, 2)).astype(F))
    x[..., 1] = np.where(x[..., 1] < 0, F(-1.0), x[..., 1])
    check_all(x)
    lo, hi = ork.indicators(x)
    assert lo[..., 1].mean() > 0.2                       # the tie at -1 sits below the quantile as a whole


def test_hmc_history_against_oracle():
    check_all(hmc_history(400, 64, 6))


def test_large_column():
    """One column of n = 2^23 pooled draws: 2048 sort tiles."""
    rs = np.random.default_rng(9)
    x = (rs.standard_normal((2048, 4096, 1)) * 0.1).round(2).astype(F)   # heavily tied
    check_all(x, exact_order=False)


def test_nan_column_leaves_neighbours_unchanged():
    rs = np.random.default_rng(10)
    x = ar1(rs, 200, 16, 5)
    tgt = T.StdNormal(5)
    clean = [npy(f(tf(x), tgt)) for f in (bj.rhat, bj.ess_bulk, bj.ess_tail)]
    x[17, 3, 2] = np.nan
    check_all(x)
    dirty = [npy(f(tf(x), tgt)) for f in (bj.rhat, bj.ess_bulk, bj.ess_tail)]
    for c, d in zip(clean, dirty):
        assert np.isnan(d[2])
    keep = [0, 1, 3, 4]
    np.testing.assert_array_equal(dirty[0][keep], clean[0][keep])
    for c, d in zip(clean[1:], dirty[1:]):
        ess_rule(d[keep], c[keep])


@pytest.mark.parametrize("shape", [(200, 16, 70), (101, 4, 9)])
def test_chunking_is_invisible(shape):
    T_, C, D = shape
    rs = np.random.default_rng(12)
    x = special(rs, T_, C, D)
    hx, tgt = tf(x), T.StdNormal(D)
    one = int(_lib.lib().bjx_rank_diagnostics_scratch_bytes(T_, C, D, 1))
    for folded in (False, True):
        a = bj.diagnostics.rank_normalize(hx, tgt, folded=folded, max_scratch_bytes=one)
        b = bj.diagnostics.rank_normalize(hx, tgt, folded=folded)
        assert torch.equal(a, b)
    assert torch.equal(bj.rhat(hx, tgt, max_scratch_bytes=one), bj.rhat(hx, tgt))
    ess_rule(npy(bj.ess_bulk(hx, tgt, max_scratch_bytes=one)), npy(bj.ess_bulk(hx, tgt)))
    ess_rule(npy(bj.ess_tail(hx, tgt, max_scratch_bytes=one)), npy(bj.ess_tail(hx, tgt)))


def test_reference_recipes_on_device_histories():
    gen = torch.Generator(DEV).manual_seed(3)
    C, T_, D = 4, 2000, 3
    tgt = T.StdNormal(D)
    iid = torch.randn(T_, C, D, device=DEV, generator=gen)
    assert np.all(np.abs(npy(bj.rhat(iid, tgt)) - 1.0) < 0.01)
    shifted = iid.clone()
    shifted[:, 3] += 3.0
    assert np.all(npy(bj.rhat(shifted, tgt)) > 1.1)
    scaled = iid.clone()
    scaled[:, 3] *= 4.0
    assert np.all(npy(bj.rhat(scaled, tgt)) > 1.05)
    e = npy(bj.ess_bulk(iid, tgt))
    assert np.all((e > 0.5 * C * T_) & (e < 2 * C * T_))
    t = npy(bj.ess_tail(iid, tgt))
    ar = tf(ar1(np.random.default_rng(4), T_, C, D))
    phi = np.linspace(-0.6, 0.95, D)
    slow = phi > 0.5
    assert np.all(npy(bj.ess_bulk(ar, tgt))[slow] < 0.5 * e[slow])
    assert np.all(npy(bj.ess_tail(ar, tgt))[slow] < t[slow])


def test_top_level_api():
    assert bj.rhat is bj.diagnostics.rhat
    assert bj.ess_bulk is bj.diagnostics.ess_bulk
    assert bj.ess_tail is bj.diagnostics.ess_tail
    assert bj.ess is bj.diagnostics.effective_sample_size


def test_rejections():
    tgt = T.StdNormal(3)
    x = torch.randn(3, 4, 3, device=DEV)
    for f in (bj.rhat, bj.ess_bulk, bj.ess_tail):
        with pytest.raises(BjxError, match="num_samples >= 4"):
            f(x, tgt)
    with pytest.raises(BjxError, match="num_samples >= 4"):
        bj.diagnostics.rank_normalize(x, tgt)
    x = torch.randn(8, 4, 3, device=DEV)
    for prob in (0.0, 1.0, -0.5, 1.5, float("nan"), float("inf")):
        with pytest.raises(BjxError, match=r"prob must be finite and in \(0, 1\)"):
            bj.ess_tail(x, tgt, prob=prob)
    with pytest.raises(BjxError, match=r"scratch too small: one dimension per pass needs \d+ bytes"):
        bj.rhat(x, tgt, max_scratch_bytes=1000)
    # n = 2C * (T // 2) >= 2^31: rejected before the history is read
    eng = get_engine(x[0], tgt)
    L = _lib.lib()
    out = torch.empty(3, device=DEV)
    scratch = torch.empty(1 << 20, dtype=torch.uint8, device=DEV)
    big_t = (1 << 29) + 2
    rc = L.bjx_rank_diagnostics(eng.h, ptr(x), big_t, 0.9, ptr(out), None, None, ptr(scratch), scratch.numel())
    with pytest.raises(BjxError, match=r"< 2\^31"):
        check(rc, eng.h)
    rc = L.bjx_rank_normalize(eng.h, ptr(x), big_t, 0, ptr(out), ptr(scratch), scratch.numel())
    with pytest.raises(BjxError, match=r"< 2\^31"):
        check(rc, eng.h)
