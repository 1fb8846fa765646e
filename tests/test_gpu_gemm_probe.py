"""The dense-path product bjx::k_gemm_f16x3 (bjx_gemm.cu), called directly, against float64 and against the exact host
models of oracle/gemm_f16x3.py.

tests/csrc/libgemm_probe.so (built by build()) is a C entry point into bjx::gemm_f16x3 of the shipped libbjx.so, so any
shape and epilogue that bjx_gemm.h allows can be run, not only the ones the samplers use.  The tile counts
ceil(M / 128) ceil(N / 128) are chosen against the device's SM count (one persistent CTA per SM): one tile, one wave
minus, exactly and plus one tile, two waves and two plus one, and about ten waves, where each CTA runs a tile's
epilogue in slices under the next tile's K loop.  K covers fewer, as many and more 64-deep K blocks than the 16
epilogue slices.

  a. the product against float64 over the operand planes, random-sign and same-sign data, K up to 18432;
  b. every epilogue mode bit for bit against the host model applied to the kernel's own accumulator (plain mode with
     alpha = 1 writes the raw accumulator; the K loop does not depend on the mode);
  c. the emitted planes, their unscales, the row maxima and the cleared next accumulator, bit for bit;
  d. nothing written before or after Y, the planes and the per-row arrays, nor in the plane pads [N, KP_out);
  e. a row's output does not depend on which tile, CTA or wave computes it;
  f. the emitted planes at the edges of the exact lift window [2^-3, 2^15.5) reconstruct Y to 2^-22 of the row maximum;
  g. a NaN or inf in one row leaves every other row's bits as they were.
"""
import ctypes
import math
import os
import sys
import zlib

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import gemm_f16x3 as G  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PROBE_PATH = os.path.join(ROOT, "tests", "csrc", "libgemm_probe.so")
F32, F64 = torch.float32, torch.float64
PAD = 64                      # guard elements before and after every output (keeps the views 16-byte aligned)
SENT32 = 0x7FA5A5A5           # a NaN payload no kernel produces
SENT16 = -0x5A5B              # 0xA5A5
_probe = None


def probe():
    global _probe
    if _probe is None:
        if not os.path.exists(PROBE_PATH):
            pytest.fail(f"{PROBE_PATH} has not been built: run __graft_entry__.build() (make -C tests/csrc)")
        from blackjax_b200 import _lib
        _lib.lib()  # the library the probe links against, loaded once
        lib = ctypes.CDLL(PROBE_PATH)
        fn = lib.bjx_probe_gemm_f16x3
        vp, i, f = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
        fn.argtypes = [vp] * 5 + [i] * 5 + [f, vp, vp, vp, f, i, i, i, vp, vp, vp, vp, vp]
        fn.restype = i
        _probe = fn
    return _probe


def sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def n_tiles(M, N):
    return -(-M // 128) * -(-N // 128)


def _ptr(t):
    return None if t is None else t.data_ptr()


def guarded(n, dtype, fill):
    full = torch.full((n + 2 * PAD,), fill, dtype=dtype, device=DEV)
    return full, full[PAD:PAD + n]


def _bits(t):
    return t.contiguous().view(torch.int32 if t.element_size() == 4 else torch.int16)


def assert_bits(got, want, what):
    """Equal bits, any NaN matching any NaN."""
    g, w = _bits(got), _bits(want)
    fg = got.contiguous().view(F32 if got.element_size() == 4 else torch.float16)
    fw = want.contiguous().view(F32 if want.element_size() == 4 else torch.float16)
    bad = (g != w) & ~(torch.isnan(fg) & torch.isnan(fw))
    if bad.any():
        idx = bad.nonzero()[:4].tolist()
        ex = [(tuple(ix), fg[tuple(ix)].item(), fw[tuple(ix)].item()) for ix in idx]
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} differ, e.g. (index, kernel, model) {ex}")


class Operands:
    """X [M, K] and A [N, K] on the device and their operand planes as k_rows_split2 / k_matrix_split2 make them."""

    def __init__(self, M, N, K, seed, same_sign=False, row_scales=True, X=None):
        g = torch.Generator(device=DEV).manual_seed(seed)
        self.M, self.N, self.K, self.KP = M, N, K, G.plane_stride(K)
        if X is None:
            X = torch.randn(M, K, generator=g, device=DEV)
            if row_scales:
                X = X * torch.pow(10.0, torch.empty(M, 1, device=DEV).uniform_(-6, 6, generator=g))
        A = torch.randn(N, K, generator=g, device=DEV)
        if same_sign:
            X, A = X.abs(), A.abs()
        self.X, self.A = X.to(F32), A.to(F32)
        self.xp, self.xu = G.rows_split2(self.X)
        self.ap, self.au = G.matrix_split2(self.A)
        self.gen = g

    def rand(self, *shape, lo=-1.0, hi=1.0):
        return torch.empty(*shape, device=DEV).uniform_(lo, hi, generator=self.gen)


def launch(op, *, alpha=1.0, alpha_dev=None, x_unscale=None, mat_unscale=None, beta=0.0, cin=None, cin_alias=False,
           double_kick=False, planes=False, stale_max=None, KP_out=None, xp=None):
    """One product through the probe, every output inside sentinel guards; checks the guards and returns the outputs."""
    M, N = op.M, op.N
    KPo = KP_out or G.plane_stride(N)
    yfull, y = guarded(M * N, torch.int32, SENT32)
    y = y.view(F32)
    cin_t = None
    if cin is not None:
        if cin_alias:
            y.copy_(cin.reshape(-1))
            cin_t = y
        else:
            cin_t = cin.contiguous()
    pfull, pl = guarded(M * 2 * KPo, torch.int16, SENT16)
    oufull, ou = guarded(M, torch.int32, SENT32)
    nmfull, nm = guarded(M, torch.int32, SENT32)
    zmfull, zm = guarded(M, torch.int32, SENT32)
    nm.zero_()  # this production's maxima accumulate from zero
    stream = torch.cuda.current_stream(DEV).cuda_stream
    rc = probe()(_ptr(op.xp if xp is None else xp), _ptr(op.ap), _ptr(y), _ptr(cin_t), _ptr(pl) if planes else None,
                 M, N, op.K, op.KP, KPo, float(alpha), _ptr(alpha_dev), _ptr(x_unscale), _ptr(mat_unscale), float(beta),
                 int(cin is not None), int(double_kick), int(planes), _ptr(ou) if planes else None,
                 _ptr(stale_max) if planes else None, _ptr(nm) if planes else None, _ptr(zm) if planes else None,
                 stream)
    assert rc == 0, f"gemm_f16x3 returned {rc}"
    torch.cuda.synchronize()
    for name, full, n in (("Y", yfull, M * N), ("planes", pfull, M * 2 * KPo), ("out_unscale", oufull, M),
                          ("next_max", nmfull, M), ("zero_max", zmfull, M)):
        fill = SENT16 if name == "planes" else SENT32
        assert bool((full[:PAD] == fill).all()), f"{name}: written before its first element"
        assert bool((full[PAD + n:] == fill).all()), f"{name}: written past its last element"
    pl = pl.view(M, 2, KPo)
    if planes:
        assert bool((pl[:, :, N:] == SENT16).all()), "planes: written in the pads [N, KP_out)"
    else:
        assert bool((pl == SENT16).all()) and bool((ou == SENT32).all()) and bool((nm == 0).all()), \
            "planes / per-row outputs written with planes = 0"
    return dict(Y=y.view(M, N), planes=pl, out_unscale=ou.view(F32), next_max=nm.view(F32), zero_max=zm.view(F32))


def acc_of(op, xp=None):
    """The kernel's raw float32 accumulator: plain mode, alpha = 1, no unscales, no Cin."""
    return launch(op, xp=xp)["Y"].clone()


# ---- shapes --------------------------------------------------------------------------------------------------
def multi_tile_shapes():
    """(name, M, N, K) with tile counts placed against the SM count S."""
    S = sms()
    return [
        ("1tile_tail20_n4_k132", 20, 4, 132),
        ("Sm1_tail1_n128_k1028", 128 * (S - 2) + 1, 128, 1028),
        ("S_n4_k4100", 128 * S, 4, 4100),
        ("Sp1_tail20_n124_k196", 128 * S + 20, 124, 196),
        ("Sp2_tail127_n132_k1024", 128 * (S // 2) + 127, 132, 1024),
        ("2S_tail127_n256_k1024", 128 * (S - 1) + 127, 256, 1024),
        ("2Sp1_tail1_n128_k1020", 128 * 2 * S + 1, 128, 1020),
        ("129rows_n260_k1020", 129, 260, 1020),
        ("about2S_tail1_n644_k1028", 128 * (S // 3) + 1, 644, 1028),
        ("about10S_tail127_n1028_k132", 128 * (-(-10 * S // 9) - 1) + 127, 1028, 132),
        ("about10S_tail20_n1024_k196", 128 * (-(-10 * S // 8) - 1) + 20, 1024, 196),
    ]


SHAPE_IDS = ["1tile_tail20_n4_k132", "Sm1_tail1_n128_k1028", "S_n4_k4100", "Sp1_tail20_n124_k196",
             "Sp2_tail127_n132_k1024", "2S_tail127_n256_k1024", "2Sp1_tail1_n128_k1020", "129rows_n260_k1020",
             "about2S_tail1_n644_k1028", "about10S_tail127_n1028_k132", "about10S_tail20_n1024_k196"]
_cache = {}


def shape_case(name):
    """The operands of a named shape and the kernel's accumulator for them, built once per module."""
    if name not in _cache:
        _cache.clear()
        (_, M, N, K), = [s for s in multi_tile_shapes() if s[0] == name]
        op = Operands(M, N, K, seed=zlib.crc32(name.encode()))
        _cache[name] = (op, acc_of(op))
    return _cache[name]


def per_row_inputs(op):
    """Per-row epilogue inputs that differ from row to row: step sizes with zero, negative and huge entries,
    power-of-two unscales, and stale maxima with zero / non-finite entries."""
    M = op.M
    ad = op.rand(M, lo=-2.0, hi=2.0)
    ad[0::11] = 0.0
    ad[5::13] = -3.5
    ad[7::17] = 1.0e30
    xu = torch.pow(2.0, torch.randint(-20, 20, (M,), device=DEV, generator=op.gen).float())
    mu = torch.tensor([2.0 ** -9], device=DEV)
    stale = (op.rand(M, lo=0.5, hi=1.0) * torch.pow(2.0, torch.randint(-30, 30, (M,), device=DEV,
                                                                      generator=op.gen).float()))
    stale[3::19] = 0.0
    stale[9::23] = float("inf")
    stale[10::29] = float("nan")
    cin = op.rand(M, op.N, lo=-1.0, hi=1.0) * torch.pow(2.0, torch.randint(-10, 10, (M, 1), device=DEV,
                                                                         generator=op.gen).float())
    return ad, xu, mu, stale, cin


# ---- a. accuracy against float64 ------------------------------------------------------------------------------
ACC_K = [132, 196, 1020, 1024, 1028, 4100, 18432]
# max over rows of max |Y - (x1 + x2)(a1 + a2)^T| / max |row of the reference|, (random-sign, same-sign), measured on
# an H100 80GB HBM3 (700 W power limit) with the data of _accuracy.  The error grows about linearly in K (the tensor
# core's float32 accumulation; ~6e-9 K random-sign, ~9e-9 K same-sign): 1e-5 holds up to K = 1028 for random-sign data.
MEASURED = {132: (1.456e-6, 2.000e-6), 196: (1.899e-6, 2.352e-6), 1020: (6.449e-6, 1.005e-5),
            1024: (6.436e-6, 9.781e-6), 1028: (6.424e-6, 1.014e-5), 4100: (2.469e-5, 3.769e-5),
            18432: (9.999e-5, 1.622e-4)}


def _accuracy(K, same_sign):
    M, N = (128, 132) if K == 18432 else (640, 260)
    op = Operands(M, N, K, seed=K + same_sign, same_sign=same_sign)
    y = acc_of(op).double()
    ref = G.planes_value(op.xp, K) @ G.planes_value(op.ap, K).T
    err = ((y - ref).abs().amax(1) / ref.abs().amax(1)).max().item()
    return err


def test_product_accuracy_against_float64():
    rows = []
    for K in ACC_K:
        rows.append((K, _accuracy(K, False), _accuracy(K, True)))
    print("\n   K   random-sign   same-sign   (max error relative to the row maximum)")
    for K, r, s in rows:
        print(f"{K:6d}   {r:.3e}    {s:.3e}")
    for K, r, s in rows:
        assert K > 1028 or r <= 1e-5, f"K = {K}: random-sign error {r:.3e} relative to the row maximum"
        assert r <= 1.5 * MEASURED[K][0], f"K = {K}: random-sign error {r:.3e} above 1.5x the measured bound"
        assert s <= 1.5 * MEASURED[K][1], f"K = {K}: same-sign error {s:.3e} above 1.5x the measured bound"


# ---- b. every epilogue mode, bit for bit ----------------------------------------------------------------------
@pytest.mark.parametrize("name", SHAPE_IDS)
def test_epilogue_modes_bit_exact(name):
    op, acc = shape_case(name)
    ad, xu, mu, stale, cin = per_row_inputs(op)
    modes = {
        "scalar alpha, unscales": dict(alpha=-0.37, x_unscale=xu, mat_unscale=mu),
        "scalar alpha only": dict(alpha=3.0e-3),
        "per-row alpha, unscales": dict(alpha=0.81, alpha_dev=ad, x_unscale=xu, mat_unscale=mu),
        "beta Cin": dict(alpha=0.5, alpha_dev=ad, x_unscale=xu, beta=-0.75, cin=cin),
        "beta Cin, Cin aliasing Y": dict(alpha=1.0, alpha_dev=ad, mat_unscale=mu, beta=1.0, cin=cin, cin_alias=True),
        "double kick": dict(alpha=-0.5, alpha_dev=ad, x_unscale=xu, mat_unscale=mu, beta=1.0, cin=cin,
                            double_kick=True),
        "planes": dict(alpha=1.0, alpha_dev=ad, x_unscale=xu, beta=1.0, cin=cin, planes=True, stale_max=stale),
        "planes, double kick, wide pads": dict(alpha=-0.5, alpha_dev=ad, x_unscale=xu, mat_unscale=mu, beta=1.0,
                                               cin=cin, double_kick=True, planes=True, stale_max=stale,
                                               KP_out=G.plane_stride(op.N) + 24),
    }
    for mode, kw in modes.items():
        out = launch(op, **kw)
        model_kw = {k: kw[k] for k in ("alpha", "alpha_dev", "x_unscale", "mat_unscale", "beta", "cin",
                                       "double_kick") if k in kw}
        want = G.epilogue(acc, **model_kw)
        assert_bits(out["Y"], want, f"{name} / {mode}: Y")


# ---- c. emitted state ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SHAPE_IDS)
def test_emitted_planes_and_row_maxima_bit_exact(name):
    op, acc = shape_case(name)
    ad, xu, mu, stale, cin = per_row_inputs(op)
    for double_kick in (False, True):
        KPo = G.plane_stride(op.N) + (8 if double_kick else 0)
        out = launch(op, alpha=0.5, alpha_dev=ad, x_unscale=xu, mat_unscale=mu, beta=1.0, cin=cin,
                     double_kick=double_kick, planes=True, stale_max=stale, KP_out=KPo)
        y = out["Y"]
        planes, unscale = G.emitted_planes(y, stale, KPo)
        what = f"{name} (double kick {double_kick})"
        assert_bits(out["planes"][:, :, :op.N], planes[:, :, :op.N], f"{what}: planes")
        assert_bits(out["out_unscale"], unscale, f"{what}: out_unscale")
        assert_bits(out["next_max"], G.row_max(y), f"{what}: next_max")
        assert bool((_bits(out["zero_max"]) == 0).all()), f"{what}: zero_max not cleared for every row"


# ---- d. out-of-bounds writes -----------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["1tile_tail20_n4_k132", "Sp1_tail20_n124_k196", "about2S_tail1_n644_k1028"])
def test_no_writes_out_of_bounds(name):
    """launch() checks the guards before and after Y, the planes and the per-row arrays, and the plane pads, on every
    call; here with pads as wide as a whole 64-column K block and with planes off (nothing but Y written)."""
    op, _ = shape_case(name)
    ad, xu, mu, stale, cin = per_row_inputs(op)
    launch(op, alpha=1.0, alpha_dev=ad, beta=1.0, cin=cin, planes=True, stale_max=stale,
           KP_out=G.plane_stride(op.N) + 64)
    launch(op, alpha=1.0, alpha_dev=ad, beta=1.0, cin=cin, double_kick=True)


# ---- e. row position ----------------------------------------------------------------------------------------------
def test_row_permutation_within_a_tile():
    op = Operands(128, 260, 1028, seed=11)
    base = acc_of(op)
    perm = torch.randperm(128, device=DEV, generator=op.gen)
    got = acc_of(op, xp=op.xp[perm].contiguous())
    assert_bits(got, base[perm], "rows permuted inside one tile")


@pytest.mark.parametrize("N, K", [(260, 1028), (128, 196)])
def test_row_position_does_not_matter(N, K):
    """Copies of one 128-row block at every row block of a multi-tile shape (a CTA's first, second and last tile,
    the partial last wave, the M tail) equal the block run alone, with every epilogue input copied along."""
    S = sms()
    tn = -(-N // 128)
    M = 128 * (-(-(2 * S + S // 2) // tn)) + 20
    assert n_tiles(M, N) > 2 * S and n_tiles(M, N) % S != 0
    base = Operands(128, N, K, seed=N + K)
    ad, xu, mu, stale, cin = per_row_inputs(base)
    kw = dict(alpha=0.5, mat_unscale=mu, beta=1.0, double_kick=True, planes=True)
    want = launch(base, alpha_dev=ad, x_unscale=xu, cin=cin, stale_max=stale, **kw)
    reps = -(-M // 128)
    idx = torch.arange(M, device=DEV) % 128
    big = Operands(M, N, K, seed=0, X=base.X[idx])
    big.A, big.ap, big.au = base.A, base.ap, base.au
    assert_bits(big.xp, base.xp[idx], "copied operand planes")
    got = launch(big, alpha_dev=ad[idx], x_unscale=xu[idx], cin=cin[idx], stale_max=stale[idx], **kw)
    for key in ("Y", "planes", "out_unscale", "next_max"):
        for b in range(reps):
            rows = slice(128 * b, min(M, 128 * b + 128))
            n = rows.stop - rows.start
            assert_bits(got[key][rows], want[key][:n], f"{key}, copy at rows {rows.start}..{rows.stop}")


# ---- f. the lift window's edges -----------------------------------------------------------------------------------
def test_lift_window_edges_reconstruct():
    """Rows whose maximum lands, after the stale lift, exactly on 2^-3, one ulp above it, just below 2^15.5 (the
    largest float32 the window test accepts) or in the middle of the window: the emitted planes reconstruct Y to
    2^-22 of the row maximum (bjx_gemm.h), the claim k_planes_fixup relies on for the rows it leaves alone."""
    S = sms()
    op = Operands(128 * S + 20, 260, 196, seed=5)
    op.A[0] = 0.0                                  # column 0 of the product is exactly zero: y[:, 0] = Cin[:, 0]
    op.ap, op.au = G.matrix_split2(op.A)
    acc = acc_of(op)
    M = op.M
    edges = torch.tensor([0.125, float(np.nextafter(np.float32(0.125), np.float32(1))),
                          float(np.nextafter(np.float32(G.PLANE_WINDOW_HI), np.float32(0))), 1.0], device=DEV)
    t = edges[torch.arange(M, device=DEV) % 4]
    s = torch.randint(-20, 21, (M,), device=DEV, generator=op.gen).float()
    stale = 1.5 * torch.pow(2.0, 6.0 - s)          # plane_lift(stale) = 2^s
    assert bool((G.plane_lift(stale) == torch.pow(2.0, s)).all())
    m = t * torch.pow(2.0, -s)                     # the row maximum, lifted to t
    cin = torch.zeros(M, op.N, device=DEV)
    cin[:, 0] = m
    # the product part stays below m / 4: a power of two per row
    amax = acc.abs().amax(1).clamp_min(1e-30)
    ad = torch.pow(2.0, torch.floor(torch.log2(m / amax)) - 2)
    out = launch(op, alpha=1.0, alpha_dev=ad, beta=1.0, cin=cin, planes=True, stale_max=stale)
    y = out["Y"]
    assert_bits(out["next_max"], m, "row maxima")
    assert_bits(out["next_max"] * G.plane_lift(stale), t, "lifted row maxima")
    planes, unscale = G.emitted_planes(y, stale, G.plane_stride(op.N))
    assert_bits(out["planes"][:, :, :op.N], planes[:, :, :op.N], "planes")
    rec = G.planes_value(out["planes"], op.N) * out["out_unscale"].double()[:, None]
    err = (rec - y.double()).abs().amax(1) / m.double()
    for i, name in enumerate(["2^-3", "one ulp above 2^-3", "just below 2^15.5", "1"]):
        e = err[i::4].max().item()
        assert e <= 2.0 ** -22, f"lifted maximum {name}: reconstruction error {e:.3e} of the row maximum > 2^-22"


# ---- g. non-finite rows ----------------------------------------------------------------------------------------------
def test_non_finite_rows_stay_in_their_rows():
    S = sms()
    op = Operands(128 * S + 20, 260, 1028, seed=9)
    ad, xu, mu, stale, cin = per_row_inputs(op)
    kw = dict(alpha=0.5, alpha_dev=ad, mat_unscale=mu, beta=1.0, planes=True, stale_max=stale)
    clean = launch(op, x_unscale=op.xu, cin=cin, **kw)
    M = op.M
    r_xnan, r_xinf, r_cnan, r_cinf = 300, 128 * S + 3, 4, M - 1
    X = op.X.clone()
    X[r_xnan, 17] = float("nan")
    X[r_xinf, 1000] = float("inf")
    xp, xu2 = G.rows_split2(X)
    cin2 = cin.clone()
    cin2[r_cnan, 130] = float("nan")
    cin2[r_cinf, 259] = -float("inf")
    dirty = launch(op, xp=xp, x_unscale=xu2, cin=cin2, **kw)
    poisoned = torch.tensor([r_xnan, r_xinf, r_cnan, r_cinf], device=DEV)
    keep = torch.ones(M, dtype=torch.bool, device=DEV)
    keep[poisoned] = False
    for key in ("Y", "planes", "out_unscale", "next_max"):
        assert_bits(dirty[key][keep], clean[key][keep], f"{key} of the clean rows")
    y = dirty["Y"]
    assert bool(torch.isnan(y[r_xnan]).all()) and bool(torch.isnan(y[r_xinf]).all())
    assert int(torch.isnan(y[r_cnan]).sum()) == 1 and bool(torch.isnan(y[r_cnan, 130]))
    assert y[r_cinf, 259].item() == -float("inf") and bool(torch.isfinite(y[r_cinf, :259]).all())
    nm = dirty["next_max"]
    assert_bits(nm[poisoned], G.row_max(y[poisoned]), "next_max of the poisoned rows")
    assert nm[r_xnan].item() == 0.0 and nm[r_cinf].item() == float("inf")
    assert math.isfinite(nm[r_cnan].item()) and nm[r_cnan].item() > 0
    assert bool((_bits(dirty["zero_max"]) == 0).all())
