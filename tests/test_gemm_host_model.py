"""The host models of the dense-path product (oracle/gemm_f16x3.py) against hand-worked cases and exact arithmetic.

tests/test_gpu_gemm_probe.py compares the kernel with these models bit for bit, so the models themselves must be exact:
the lifts mirror bjx::pow2_lift_to including its clamps and non-finite cases, the plane split rounds like
__float2half_rn (checked against numpy's binary16 conversion), and the float32 fmaf emulation is checked against
fractions.Fraction on ties, cancellations and wide exponent gaps.
"""
import os
import sys
from fractions import Fraction

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import gemm_f16x3 as G  # noqa: E402

F32 = np.float32


def _t(a):
    return torch.from_numpy(np.asarray(a, F32))


def test_pow2_lift_hand_cases():
    tiny = np.float32(1e-45)                     # the smallest subnormal, exponent field 0
    cases = [  # (amax, e, expected lift)
        (0.0, 13, 1.0), (-0.0, 13, 1.0), (-5.0, 13, 1.0), (np.nan, 13, 1.0), (np.inf, 13, 1.0), (3.1e38, 13, 1.0),
        (3.0e38, 13, 2.0 ** (13 - 127)),         # not above 3e38: lifted (down) like any other maximum
        (1.0, 13, 2.0 ** 13), (1.5, 13, 2.0 ** 13), (np.nextafter(F32(2), F32(0)), 13, 2.0 ** 13),
        (2.0, 13, 2.0 ** 12), (2.0 ** 13, 13, 1.0), (2.0 ** 14, 13, 0.5), (0.75, 6, 2.0 ** 7),
        (2.0 ** -126, 6, 2.0 ** 126),            # 6 + 126 = 132 clamps at +126
        (tiny, 6, 2.0 ** 126), (np.float32(2.0 ** -140), 13, 2.0 ** 126),  # subnormals: exponent field 0 -> s = e + 127
        (2.0 ** 127, 6, 2.0 ** -121), (2.0 ** 127, -10, 2.0 ** -126),      # 2^-137 clamps at -126
        (2.0 ** 100, -40, 2.0 ** -126),
    ]
    a = _t([c[0] for c in cases])
    for e in sorted({c[1] for c in cases}):
        sel = [i for i, c in enumerate(cases) if c[1] == e]
        got = G.pow2_lift_to(a[sel], e).numpy()
        want = np.array([cases[i][2] for i in sel], F32)
        assert np.array_equal(got.view(np.int32), want.view(np.int32)), (e, a[sel], got, want)
    # the named lifts and their targets: every finite positive maximum in the normal range lands in [2^e, 2^(e+1))
    m = np.float32(2.0) ** np.arange(-100, 100, dtype=F32) * np.float32(1.37)
    for fn, e in ((G.pow2_lift, 13), (G.plane_lift, 6)):
        lifted = m * fn(_t(m)).numpy()
        assert np.all((lifted >= 2.0 ** e) & (lifted < 2.0 ** (e + 1)))


def test_split_matches_numpy_binary16():
    rs = np.random.default_rng(1)
    y = (rs.standard_normal((64, 300)) * np.exp2(rs.integers(-30, 30, (64, 1)))).astype(F32)
    y[0, :4] = [0.0, -0.0, 65519.0 / 2 ** 6, 2.0 ** -30]
    y[1, :3] = [np.inf, -np.inf, np.nan]
    sc = np.exp2(rs.integers(-20, 20, 64)).astype(F32)
    got = G.split_planes(_t(y), _t(sc), 304).numpy().view(np.uint16)
    with np.errstate(over="ignore", invalid="ignore"):
        s = y * sc[:, None]
        h1 = s.astype(np.float16)
        h2 = (s - h1.astype(F32)).astype(np.float16)
    assert np.array_equal(got[:, 0, :300], h1.view(np.uint16))
    assert np.array_equal(got[:, 1, :300], h2.view(np.uint16))
    assert not got[:, :, 300:].any()
    # the exact split of a row reconstructs it to 2^-22 of its maximum
    planes, unscale = G.rows_split2(_t(y[2:]))
    err = (G.planes_value(planes, 300) * unscale.double()[:, None] - torch.from_numpy(y[2:]).double()).abs()
    assert torch.all(err <= 2.0 ** -22 * torch.from_numpy(np.abs(y[2:])).double().amax(1, keepdim=True))


def _round_fraction_to_f32(x):
    """The float32 nearest to the rational x, ties to even; +-inf past the overflow threshold."""
    if x == 0:
        return 0.0
    neg = x < 0
    x = -x if neg else x
    e = x.numerator.bit_length() - x.denominator.bit_length()
    if Fraction(2) ** e > x:
        e -= 1
    q = Fraction(2) ** (max(e, -126) - 23)   # the float32 spacing at x
    n = x / q
    m = n.numerator // n.denominator
    rem = n - m
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and m % 2 == 1):
        m += 1
    v = m * q
    r = float("inf") if v >= Fraction(2) ** 128 else float(v)
    return -r if neg else r


def _fma_samples(rs, n):
    """float32 triples (a, b, c) of five kinds: random, halfway ties with and without a tiny term past float64's
    reach, cancellation, and wide exponent gaps."""
    def f32(v):
        return np.asarray(v, F32)

    k = n // 5
    out = []
    # 1. random significands and exponents over the whole normal range of the product
    a = f32(rs.standard_normal(k) * np.exp2(rs.integers(-60, 60, k)))
    b = f32(rs.standard_normal(k) * np.exp2(rs.integers(-60, 60, k)))
    c = f32(rs.standard_normal(k) * np.exp2(rs.integers(-120, 120, k)))
    out.append((a, b, c))
    # 2. products exactly halfway between two float32 (a short significand times a 24-bit one), c = 0 or a term far
    #    below float64's precision of the product: float64 rounds the sum onto the halfway point
    a = f32(rs.choice([3.0, 5.0, 7.0, 11.0, 13.0], k) * np.exp2(rs.integers(-20, 20, k)))
    b = f32((1.0 + rs.integers(1, 2 ** 23, k) * 2.0 ** -23) * np.exp2(rs.integers(-20, 20, k)))
    p = a.astype(np.float64) * b.astype(np.float64)
    tiny = np.exp2(np.floor(np.log2(np.abs(p))) - rs.integers(60, 90, k)) * rs.choice([-1.0, 0.0, 1.0], k)
    out.append((a, b, f32(tiny)))
    # 3. c = +-half an ulp of an exact float32 product (a tie of the exact sum), and that plus a tiny nudge
    a = f32(rs.integers(1, 2 ** 12, k) * np.exp2(rs.integers(-20, 20, k)))
    b = f32(rs.integers(1, 2 ** 12, k) * np.exp2(rs.integers(-20, 20, k)))
    pf = (a * b).astype(F32)
    half = (np.nextafter(pf, np.float32(np.inf)) - pf) * np.float32(0.5)
    c = f32(half * rs.choice([-1.0, 1.0], k) * (1.0 + rs.choice([0.0, 2.0 ** -23, -2.0 ** -24], k)))
    out.append((a, b, c))
    # 4. cancellation: c close to -a b
    a = f32(rs.standard_normal(k) * np.exp2(rs.integers(-30, 30, k)))
    b = f32(rs.standard_normal(k) * np.exp2(rs.integers(-30, 30, k)))
    c = f32(-(a.astype(np.float64) * b) * (1.0 + rs.integers(-4, 5, k) * 2.0 ** -24))
    out.append((a, b, c))
    # 5. wide exponent gaps either way, into the subnormal range and near the overflow threshold
    a = f32(rs.standard_normal(k) * np.exp2(rs.integers(-75, 64, k)))
    b = f32(rs.standard_normal(k) * np.exp2(rs.integers(-75, 64, k)))
    c = f32(rs.standard_normal(k) * np.exp2(rs.choice([-149, -140, -126, -100, 0, 100, 126, 127], k)))
    out.append((a, b, c))
    return [np.concatenate(x) for x in zip(*out)]


def test_fmaf_matches_exact_rounding():
    rs = np.random.default_rng(7)
    with np.errstate(over="ignore"):
        a, b, c = _fma_samples(rs, 300_000)
    ok = np.isfinite(a) & np.isfinite(b) & np.isfinite(c)
    a, b, c = a[ok], b[ok], c[ok]
    got = G.fmaf(_t(a), _t(b), _t(c)).numpy()
    want = np.array([_round_fraction_to_f32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z)))
                     for x, y, z in zip(a, b, c)], F32)
    # -0 vs +0 aside (an exact zero sum), every result has the exact rounding's bits
    same = (got.view(np.int32) == want.view(np.int32)) | ((got == 0) & (want == 0))
    bad = np.flatnonzero(~same)
    assert bad.size == 0, [(a[i], b[i], c[i], got[i], want[i]) for i in bad[:5]]
    # the samples do reach the corrected case: float64 rounding lands on a float32 halfway point
    p = a.astype(np.float64) * b.astype(np.float64)
    with np.errstate(over="ignore"):
        naive = (p + c.astype(np.float64)).astype(F32)
    assert np.count_nonzero(naive.view(np.int32) != want.view(np.int32)) > 1000


def test_fmaf_non_finite():
    nan, inf = np.nan, np.inf
    a = _t([inf, 1.0, 0.0, 1.0, 3.0e38, nan])
    b = _t([1.0, inf, inf, 2.0, 10.0, 1.0])
    c = _t([-inf, 1.0, 1.0, nan, 0.0, 0.0])
    got = G.fmaf(a, b, c).numpy()
    assert np.isnan(got[0]) and got[1] == np.inf and np.isnan(got[2]) and np.isnan(got[3])
    assert got[4] == np.inf and np.isnan(got[5])


def test_row_factor_order():
    """((alpha_dev[r] * alpha) * x_unscale[r]) * mat_unscale, each product rounded to float32."""
    rs = np.random.default_rng(3)
    M = 10_000
    ad = rs.uniform(-3, 3, M).astype(F32)
    xu = np.exp2(rs.integers(-30, 30, M)).astype(F32) * F32(1.0)
    xu[::7] = rs.uniform(0.1, 10, len(xu[::7])).astype(F32)   # non-powers of two: the order shows
    mu = np.array([0.3], F32)
    alpha = F32(0.7)
    got = G.row_factor(M, float(alpha), _t(ad), _t(xu), _t(mu)).numpy()
    want = ((ad * alpha) * xu) * mu[0]
    assert np.array_equal(got.view(np.int32), want.view(np.int32))
    other = (ad * (alpha * xu)) * mu[0]
    assert np.any(other != want)  # the cases do distinguish the order
    # and the epilogue modes built on it
    acc = rs.standard_normal((M, 1)).astype(F32)
    cin = rs.standard_normal((M, 1)).astype(F32)
    y = G.epilogue(_t(acc), 0.7, _t(ad), _t(xu), _t(mu)).numpy()
    assert np.array_equal(y, want[:, None] * acc)
    y = G.epilogue(_t(acc), 0.7, _t(ad), _t(xu), _t(mu), beta=0.5, cin=_t(cin)).numpy()
    ref = [_round_fraction_to_f32(Fraction(float(w)) * Fraction(float(x)) + Fraction(float(F32(0.5) * z)))
           for w, x, z in zip(want[:500], acc[:500, 0], cin[:500, 0])]
    assert np.array_equal(y[:500, 0], np.array(ref, F32))
