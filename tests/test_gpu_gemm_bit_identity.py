"""Bit-identity of the dense path's tensor-core product (bjx::k_gemm_f16x3, bjx_gemm.cu) across kernel revisions.

Every product of the dense path goes through this kernel: v = M^-1 p (velocity), p = L^-T z (momentum draw), g = -q P
(init_state and the closing gradient of a trajectory), q <- q + eps_c (p M^-1) with the planes of q, and the double half
kick p <- p - (eps_c / 2)(q P) twice with the planes of p (leapfrog between steps).  Changes to how the kernel schedules
its loads and MMAs must leave each output bit for bit as it was, which the parity tests (tolerances against float64 or
the oracle) cannot show.  The shapes have row, column and K tails: 129 rows over two row tiles, a 200-column tile tail,
and D = 132 whose operand planes are padded to 136.

The fixture keeps the outputs small: every row of a [C, D] output is stored as a 64-bit BLAKE2b digest of its bytes, and
the [C] log-densities as they are.  A changed bit changes its row's digest, and the failure names the rows that differ.

The fixture tests/golden/gemm_f16x3_outputs.npz was recorded on an H100 80GB HBM3 at commit cb05fff, with the kernel as it
stood before its epilogue loads were hoisted above the K loop and one wgmma group was kept in flight, by building that
commit and running this file from its tree:
    python tests/test_gpu_gemm_bit_identity.py tests/golden/gemm_f16x3_outputs.npz

These fixtures show that nothing changed, not that the output is right; correctness is checked independently by
tests/test_gpu_gemm_probe.py (the kernel called directly, against float64 and bit-exact host models of every epilogue
mode) and tests/test_gpu_dense_lift_window.py (the fused leapfrog at rows that leave the planes' exact lift window).
"""
import hashlib
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from blackjax_b200 import _engine, targets as T  # noqa: E402
from oracle import prng as oprng  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(ROOT, "tests", "golden", "gemm_f16x3_outputs.npz")
# (chains, dims, per-chain step sizes)
CASES = [(129, 1024, False), (300, 200, False), (33, 132, True)]


def _spd(rs, D):
    A = rs.standard_normal((D, D))
    return (A @ A.T / D + np.eye(D)).astype(np.float32)


def case_outputs(C, D, per_chain_eps):
    """{name: float32 array} of every dense-path product kind on one seeded (C, D) problem."""
    rs = np.random.default_rng(1000 * C + D)
    prec, imm = _spd(rs, D), _spd(rs, D)
    q = (0.5 * rs.standard_normal((C, D))).astype(np.float32)
    p = rs.standard_normal((C, D)).astype(np.float32)
    eps = rs.uniform(0.02, 0.08, C).astype(np.float32) if per_chain_eps else 0.05
    keys = oprng.split(oprng.key(C + D), C)

    def dev(a):
        return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)

    eng = _engine.Engine(DEV, C, D, T.DenseGaussian(prec))
    eng.set_metric(dev(imm))
    out = {}
    out["velocity"] = eng.velocity(dev(p))
    out["momentum"] = eng.sample_momentum(dev(keys.view(np.int32)).view(torch.uint32))
    dq, dp = dev(q), dev(p)
    logp, g = eng.init_state(dq)
    out["init_logp"], out["init_grad"] = logp.clone(), g.clone()
    eng.leapfrog_(dq, dp, logp, g, dev(eps) if per_chain_eps else eps, 3)
    out["leapfrog_q"], out["leapfrog_p"], out["leapfrog_logp"], out["leapfrog_grad"] = dq, dp, logp, g
    torch.cuda.synchronize()
    res = {k: v.cpu().numpy() for k, v in out.items()}
    eng.close()
    return res


def _key(C, D, name):
    return f"c{C}_d{D}_{name}"


def fingerprint(a):
    """[C] float32 arrays as they are; [C, D] float32 arrays as one 64-bit digest of each row's bytes."""
    a = np.ascontiguousarray(a, np.float32)
    if a.ndim == 1:
        return a
    return np.array([int.from_bytes(hashlib.blake2b(row.tobytes(), digest_size=8).digest(), "little") for row in a],
                    np.uint64)


def _bits(x):
    """Bit patterns: float32 values compare by their bits (a NaN equals the same NaN, -0 differs from +0)."""
    return x.view(np.uint32) if x.dtype == np.float32 else x


@pytest.mark.parametrize("C, D, per_chain_eps", CASES)
def test_dense_products_bit_identical(C, D, per_chain_eps):
    want = np.load(GOLDEN)
    got = case_outputs(C, D, per_chain_eps)
    for name, a in got.items():
        f, b = fingerprint(a), want[_key(C, D, name)]
        assert f.shape == b.shape and f.dtype == b.dtype, name
        rows = np.flatnonzero(_bits(f) != _bits(b))
        assert rows.size == 0, f"{name}: rows {rows[:16].tolist()} ({rows.size} of {len(f)}) differ from the recorded bits"


if __name__ == "__main__":
    arrays = {}
    for C, D, per_chain_eps in CASES:
        arrays.update({_key(C, D, k): fingerprint(v) for k, v in case_outputs(C, D, per_chain_eps).items()})
    np.savez_compressed(sys.argv[1], **arrays)
    print(f"wrote {len(arrays)} arrays to {sys.argv[1]}")
