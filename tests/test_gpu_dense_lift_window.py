"""The fused leapfrog of the dense path (dense metric and dense Gaussian target, dense_leapfrog_core in bjx_dense.cu) at
rows whose maximum leaves the exact lift window of the epilogue-emitted operand planes.

The q-update and the double half kick emit the planes of their output with a lift chosen from the row maximum the
previous production of the same variable recorded; that split is exact to 2^-22 of the row maximum only while the
lifted maximum stays in [2^-3, 2^15.5) (bjx_gemm.h).  Rows that leave the window are re-split from the float32 row by
k_planes_fixup.  A stable trajectory from ordinary positions never leaves it, so the rows here are made to:

  * q0 = 0 with a tiny momentum (the stale maximum is 0, the lift 1, and q1 lands far below 2^-3);
  * q0 = 0 with a huge momentum (without the fixup, binary16 overflows and the row turns NaN);
  * q0 of scale 2^-30 with an ordinary momentum (the stale lift is 2^36);
  * p0 = float32(-(q0 / eps) M), so that q1 = q0 + eps p0 M^-1 cancels to about 2^-20 |q0|;
  * per-chain step sizes far past the stability limit, where p and q grow by more than 2^10 per half step.

With L = 1 the closing gradient g1 = -(q1 P) is computed from the planes the q-update emitted (after the fixup), so
comparing it with float64 on the kernel's own q1 checks those planes.  Power-of-two scaling of rows with a non-zero
starting position is exactly equivariant (every lift, window test and fixup decision is scale-free; a zero stale
maximum takes the lift 1 whatever the scale, so rows starting at q = 0 are left unscaled), and rows do not depend on
the batch around them, both bit for bit.
"""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from blackjax_b200 import _engine, targets as T  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F32, F64 = torch.float32, torch.float64
EPS = 0.05
DIMS = [132, 1024, 1028]
KINDS = 8   # row r is of kind r % KINDS: 0-3 leave the window as listed above, 4-7 are ordinary


def sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


class Problem:
    def __init__(self, D, seed):
        self.D = D
        self.gen = torch.Generator(device=DEV).manual_seed(seed)
        self.prec = self._spd().to(F32)
        self.imm = self._spd().to(F32)
        self.mass = torch.linalg.inv(self.imm.double())       # M, float64

    def _spd(self):
        A = torch.randn(self.D, self.D, generator=self.gen, device=DEV, dtype=F64)
        S = A @ A.T / self.D + torch.eye(self.D, device=DEV, dtype=F64)
        return 0.5 * (S + S.T)

    def engine(self, C, prec_scale=1.0, imm_scale=1.0):
        eng = _engine.Engine(DEV, C, self.D, T.DenseGaussian((self.prec * prec_scale).cpu().numpy()))
        eng.set_metric((self.imm * imm_scale).contiguous())
        return eng

    def rows(self, C, eps):
        """q0, p0 [C, D] float32 with row kind r % KINDS; eps a float or a [C] tensor."""
        D, g = self.D, self.gen
        q = 0.5 * torch.randn(C, D, generator=g, device=DEV)
        p = torch.randn(C, D, generator=g, device=DEV)
        kind = torch.arange(C, device=DEV) % KINDS
        q[kind <= 1] = 0.0
        p[kind == 0] *= 1e-9
        p[kind == 1] *= 1e7
        q[kind == 2] *= 2.0 ** -30
        e = (eps if isinstance(eps, torch.Tensor) else torch.full((C,), eps, device=DEV)).double()
        c3 = kind == 3
        p[c3] = (-(q[c3].double() / e[c3, None]) @ self.mass).to(F32)
        return q.contiguous(), p.contiguous()

    def leapfrog64(self, q, p, g, eps, L):
        """The float64 velocity Verlet of the same inputs (g the opening gradient)."""
        e = (eps if isinstance(eps, torch.Tensor) else torch.full((q.shape[0],), eps, device=DEV)).double()[:, None]
        q, p, g = q.double(), p.double(), g.double()
        P, Minv = self.prec.double(), self.imm.double()
        p = p + 0.5 * e * g
        for s in range(L):
            q = q + e * (p @ Minv)
            g = -(q @ P)
            p = p + 0.5 * e * g
            if s + 1 < L:
                p = p + 0.5 * e * g
        return q, p, g


def run(prob, q, p, g, eps, L, eng=None):
    C = q.shape[0]
    eng = eng or prob.engine(C)
    q, p, g = q.clone(), p.clone(), g.clone()
    logp = torch.zeros(C, device=DEV)
    eng.leapfrog_(q, p, logp, g, eps, L)
    torch.cuda.synchronize()
    return q, p, g, logp


def rel_err(got, ref):
    """Per row: max |got - ref| / max |ref|."""
    return (got.double() - ref).abs().amax(1) / ref.abs().amax(1).clamp_min(1e-300)


def assert_bits(got, want, what):
    a, b = got.contiguous().view(torch.int32), want.contiguous().view(torch.int32)
    bad = (a != b) & ~(torch.isnan(got) & torch.isnan(want))
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements differ, first rows " \
                                f"{sorted(set(bad.nonzero()[:, 0].tolist()))[:8]}"


# the product's own error at K <= 1028 is up to 1e-5 of the row maximum (tests/test_gpu_gemm_probe.py); a row split
# with a lift outside the window is off by about 2^-10 of its maximum, or NaN
GRAD_TOL = 2e-5


@pytest.mark.parametrize("D", DIMS)
def test_teacher_forced_gradient_from_emitted_planes(D):
    """L = 1 from g = 0: the opening kick leaves p as given, q1 is the kernel's own q-update, and the closing gradient
    is -(q1 P) from the planes that update emitted; it must match float64 on q1 in every kind of row."""
    prob = Problem(D, seed=D)
    C = 128 * (sms() + 3) + 37
    q0, p0 = prob.rows(C, EPS)
    q1, p1, g1, _ = run(prob, q0, p0, torch.zeros_like(q0), EPS, 1)
    ref = -(q1.double() @ prob.prec.double())
    err = rel_err(g1, ref)
    kind = torch.arange(C, device=DEV) % KINDS
    q1max = q1.abs().amax(1)
    # the rows do leave the window (the stale maximum of kinds 0 and 1 is 0: their lift is 1)
    assert bool((q1max[kind == 0] < 2.0 ** -3).all()) and bool((q1max[kind == 1] > 2.0 ** 15.5).all())
    assert bool((q1max[kind == 3] < 2.0 ** -12 * q0.abs().amax(1)[kind == 3]).all())
    for k in range(KINDS):
        e = err[kind == k].max().item()
        assert np.isfinite(e) and e <= GRAD_TOL, f"D = {D}, row kind {k}: closing gradient off by {e:.3e} of its row maximum"


# max error of q, p and g relative to the row maximum after 3 unstable steps, measured on an H100 80GB HBM3 (700 W):
# 7.1e-6 at D = 132, 3.5e-5 at D = 1024 and 1028
UNSTABLE_BOUND = 5e-5


@pytest.mark.parametrize("D", DIMS)
def test_unstable_step_sizes_against_float64(D):
    prob = Problem(D, seed=10 + D)
    C = 128 * (sms() + 1) + 5
    lam = torch.linalg.eigvals(prob.imm.double() @ prob.prec.double()).real.max().item()
    factor = torch.empty(C, device=DEV).uniform_(32.0, 48.0, generator=prob.gen)
    factor[::4] = 0.5                                    # stable chains beside them
    eps = (factor / np.sqrt(lam)).to(F32)
    q0, p0 = prob.rows(C, eps)
    eng = prob.engine(C)
    _, g0 = eng.init_state(q0.clone())
    q, p, g, _ = run(prob, q0, p0, g0.clone(), eps, 3, eng)
    rq, rp, rg = prob.leapfrog64(q0, p0, g0, eps, 3)
    finite_ref = (rq.abs().amax(1) < 3e38) & (rp.abs().amax(1) < 3e38) & (rg.abs().amax(1) < 3e38)
    unstable = factor > 1.0
    grown = (rp.abs().amax(1) > 2.0 ** 20 * p0.abs().amax(1).double()) & unstable
    worst, errs = [], {}
    for name, got, ref in (("q", q, rq), ("p", p, rp), ("g", g, rg)):
        errs[name] = rel_err(got[finite_ref], ref[finite_ref]).max().item()
        worst.append(f"{name} {errs[name]:.2e}")
    print(f"\nD = {D}: unstable leapfrog, {int(grown.sum())} of {int(unstable.sum())} unstable rows grew by 2^20, "
          f"max error relative to the row maximum: {', '.join(worst)}")
    assert int(grown.sum()) > 0.9 * int(unstable.sum()), "the step sizes do not make the trajectories grow"
    for name, got in (("q", q), ("p", p), ("g", g)):
        assert bool(torch.isfinite(got[finite_ref]).all()), f"{name}: non-finite rows where float64 stays finite"
        assert errs[name] <= UNSTABLE_BOUND, f"D = {D}: {name} off by {errs[name]:.3e} of its row maximum"


@pytest.mark.parametrize("D", DIMS)
def test_power_of_two_scaling_is_exact(D):
    prob = Problem(D, seed=20 + D)
    C = 128 * (sms() + 1) + 37
    eps = torch.empty(C, device=DEV).uniform_(0.03, 0.07, generator=prob.gen)
    q0, p0 = prob.rows(C, eps)
    eng = prob.engine(C)
    _, g0 = eng.init_state(q0.clone())
    k = torch.randint(-40, 41, (C, 1), device=DEV, generator=prob.gen).float()
    # rows starting at q0 = 0 are not scaled: a zero stale maximum takes the lift 1 whatever the row's scale, so
    # whether their first q planes are re-split (and with which lift) depends on the scale
    k[(torch.arange(C, device=DEV) % KINDS <= 1)] = 0.0
    s = torch.pow(2.0, k)
    base = run(prob, q0, p0, g0, eps, 3, eng)
    scaled = run(prob, q0 * s, p0 * s, g0 * s, eps, 3, eng)
    for name, a, b in zip("qpg", base[:3], scaled[:3]):
        assert_bits(b, a * s, f"D = {D}: 2^k-scaled rows, {name}")
    # the constant matrices: velocity and init_state scale with M^-1 and P
    v = eng.velocity(p0)
    _, gi = eng.init_state(q0.clone())
    for j in (-7, 5):
        e2 = prob.engine(C, prec_scale=2.0 ** j, imm_scale=2.0 ** j)
        assert_bits(e2.velocity(p0), v * 2.0 ** j, f"D = {D}: velocity with 2^{j} M^-1")
        assert_bits(e2.init_state(q0.clone())[1], gi * 2.0 ** j, f"D = {D}: gradient with 2^{j} P")
        e2.close()
    eng.close()


@pytest.mark.parametrize("D", DIMS)
def test_batch_invariance_at_multi_tile_batch(D):
    prob = Problem(D, seed=30 + D)
    q0, p0 = prob.rows(128, EPS)
    eps = torch.empty(128, device=DEV).uniform_(0.03, 0.07, generator=prob.gen)
    eng = prob.engine(128)
    _, g0 = eng.init_state(q0.clone())
    want = run(prob, q0, p0, g0, eps, 3, eng)
    C = 2 * sms() * 128 + 37
    idx = torch.arange(C, device=DEV) % 128
    big = prob.engine(C)
    got = run(prob, q0[idx], p0[idx], g0[idx], eps[idx], 3, big)
    for name, a, b in zip(("q", "p", "g", "logp"), want, got):
        assert_bits(b, a[idx], f"D = {D}: {name} of the replicas")
    # one NaN in one row leaves every other row's bits
    qn = q0[idx].clone()
    bad = C - 50
    qn[bad, 3] = float("nan")
    got2 = run(prob, qn, p0[idx], g0[idx], eps[idx], 3, big)
    keep = torch.arange(C, device=DEV) != bad
    for name, a, b in zip(("q", "p", "g", "logp"), got, got2):
        assert_bits(b[keep], a[keep], f"D = {D}: {name} beside a NaN row")
    big.close()
    eng.close()
