"""Bit-exact models of the dense-path product's host-visible arithmetic (blackjax_b200/csrc/bjx_gemm.h, bjx_gemm.cu,
bjx_dense.cu): the power-of-two lifts, the two-plane binary16 split, float32 fmaf, and the fused epilogue applied to
the kernel's own float32 accumulator.  Everything works on torch tensors on any device, so that the GPU tests can run
the models beside the kernel and the CPU test can check them against exact rational arithmetic.

The split rounds with `Tensor.to(torch.float16)`, round-to-nearest-even like `__float2half_rn`; float32 products and
differences are single torch operations (eager torch does not contract them into FMAs).
"""
import torch

F32, F64 = torch.float32, torch.float64
PLANE_WINDOW_LO = 0.125      # 2^-3     (bjx_gemm.h kPlaneWindowLo)
PLANE_WINDOW_HI = 46340.0    # ~2^15.5  (bjx_gemm.h kPlaneWindowHi)
_OVERFLOW_MID = 2.0 ** 128 - 2.0 ** 103   # halfway between FLT_MAX and 2^128


def abs_ignoring_nan(x):
    """|x| with NaN as 0: the row maxima use fmaxf, which drops a NaN operand (inf stays inf)."""
    return torch.where(torch.isnan(x), torch.zeros_like(x), x.abs())


def plane_stride(K):
    return (K + 7) & ~7


def pow2_lift_to(amax, e):
    """bjx::pow2_lift_to: the power of two 2^s, s = e - exponent(amax) clamped to [-126, 126], that lifts amax into
    [2^e, 2^(e+1)); 1 for amax that is not > 0 or is above 3e38 (zero, NaN, inf)."""
    amax = amax.to(F32)
    ex = ((amax.view(torch.int32) >> 23) & 0xFF) - 127
    s = torch.clamp(e - ex, -126, 126)
    lift = ((s + 127) << 23).to(torch.int32).view(F32)
    keep = (amax > 0) & (amax <= 3.0e38)
    return torch.where(keep, lift, torch.ones_like(lift))


def pow2_lift(amax):
    return pow2_lift_to(amax, 13)


def plane_lift(stale_max):
    return pow2_lift_to(stale_max, 6)


def split_planes(y, sc, KP):
    """The (x1 | x2) planes [R, 2, KP] (uint16 bits of binary16, zero pads) of rows y [R, K] lifted by sc [R] (or a
    scalar tensor): s = f32(y sc), x1 = f16(s), x2 = f16(f32(s - f32(x1)))."""
    R, K = y.shape
    s = y.to(F32) * sc.to(F32).reshape(-1, 1)
    h1 = s.to(torch.float16)
    h2 = (s - h1.to(F32)).to(torch.float16)
    out = torch.zeros(R, 2, KP, dtype=torch.int16, device=y.device)
    out[:, 0, :K] = h1.view(torch.int16)
    out[:, 1, :K] = h2.view(torch.int16)
    return out


def planes_value(planes, K):
    """x1 + x2 in float64 of planes [R, 2, KP]."""
    h = planes[:, :, :K].contiguous().view(torch.float16).to(F64)
    return h[:, 0] + h[:, 1]


def rows_split2(x):
    """k_rows_split2: planes of every row of x [R, K] with the exact lift (row maximum into [2^13, 2^14)) and the
    unscales 2^-s_r."""
    amax = abs_ignoring_nan(x).amax(dim=1)
    sc = pow2_lift(amax)
    return split_planes(x, sc, plane_stride(x.shape[1])), (1.0 / sc).to(F32)


def matrix_split2(a):
    """k_absmax + k_matrix_split2: planes of a constant matrix a [N, K] with one lift, and its unscale [1]."""
    sc = pow2_lift(abs_ignoring_nan(a).amax().reshape(1))
    return split_planes(a, sc.expand(a.shape[0]), plane_stride(a.shape[1])), (1.0 / sc).to(F32)


def _round_to_f32(s, err):
    """float32 nearest to s + err (float64 TwoSum pair, |err| <= ulp(s) / 2): s.to(float32) is that value except when
    s lies exactly halfway between two float32 and err != 0, where the exact sum lies on err's side of the halfway
    point."""
    r = s.to(F32)
    r64 = r.to(F64)
    up = s > r64
    other = torch.nextafter(r, torch.where(up, torch.full_like(r, float("inf")), torch.full_like(r, -float("inf"))))
    mid = torch.where(torch.isinf(r) & torch.isfinite(s), torch.sign(s) * _OVERFLOW_MID, (r64 + other.to(F64)) * 0.5)
    fix = (s == mid) & (err != 0) & torch.isfinite(s)
    # at a halfway point, RNE chose r; the exact value is on the side of err
    toward_other = (err > 0) == (other.to(F64) > r64)
    return torch.where(fix & toward_other, other, r)


def fmaf(a, b, c):
    """float32 fmaf(a, b, c), correctly rounded: the float64 product of two float32 is exact, a TwoSum with c gives the
    sum and its exact error, and _round_to_f32 corrects the one case where rounding the float64 sum is not the
    rounding of the exact sum."""
    a, b, c = (t.to(F32).to(F64) for t in torch.broadcast_tensors(a, b, c))
    p = a * b
    s = p + c
    bp = s - c
    err = (p - bp) + (c - (s - bp))
    err = torch.where(torch.isfinite(s), err, torch.zeros_like(err))
    return _round_to_f32(s, err)


def row_factor(M, alpha, alpha_dev=None, x_unscale=None, mat_unscale=None, device="cpu"):
    """The epilogue's per-row factor in the kernel's order: ((alpha_dev[r] * alpha) * x_unscale[r]) * mat_unscale."""
    al = torch.full((M,), alpha, dtype=F32, device=device)
    if alpha_dev is not None:
        al = alpha_dev.to(F32) * al
    al = al * (x_unscale.to(F32) if x_unscale is not None else torch.ones(M, dtype=F32, device=device))
    mu = mat_unscale.to(F32).reshape(1) if mat_unscale is not None else torch.ones(1, dtype=F32, device=device)
    return al * mu


def epilogue(acc, alpha=1.0, alpha_dev=None, x_unscale=None, mat_unscale=None, beta=0.0, cin=None,
             double_kick=False):
    """Y of the fused epilogue from the float32 accumulator acc [M, N]:
    lincomb y = fmaf(al, acc, f32(beta cin)); double kick y = fmaf(al, acc, fmaf(al, acc, cin)); no Cin: y = al acc."""
    M = acc.shape[0]
    al = row_factor(M, alpha, alpha_dev, x_unscale, mat_unscale, acc.device).reshape(-1, 1)
    if cin is None:
        return al * acc
    if double_kick:
        return fmaf(al, acc, fmaf(al, acc, cin))
    return fmaf(al, acc, torch.tensor(beta, dtype=F32, device=acc.device) * cin)


def row_max(y):
    """The epilogue's row maximum of |y|: NaN ignored (fmaxf), 0 for an all-NaN row."""
    return abs_ignoring_nan(y).amax(dim=1)


def emitted_planes(y, stale_max, KP_out):
    """The epilogue's planes of y [M, N] (lifted by plane_lift(stale_max)) and their unscales."""
    sc = plane_lift(stale_max)
    return split_planes(y, sc, KP_out), (1.0 / sc).to(F32)
