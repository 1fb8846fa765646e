"""Bit-identity of the dense path's tensor-core product (bjx::k_gemm_f16x3, bjx_gemm.cu) at the tail shapes that
tests/test_gpu_gemm_bit_identity.py does not cover: row and column tails of the epilogue's whole-row stores, and tile
counts that schedules tying neighbouring column tiles together (CTA clusters along N, DESIGN §9) have to handle:

  (1, 1024, True)    one live row, as in dense NUTS' compacted leaves;
  (70, 260, False)   3 column tiles, the last one 4 columns wide: an odd number of column tiles per row block;
  (129, 644, True)   6 column tiles: not a multiple of 4 column tiles per row block.

Products, inputs and fingerprints are those of tests/test_gpu_gemm_bit_identity.py, imported from it.

The fixture tests/golden/gemm_f16x3_tail_shapes.npz was recorded on an H100 80GB HBM3 with the single-CTA kernel of
commit 63c6297, by building that commit and running this file from its tree:
    python tests/test_gpu_gemm_tail_shapes.py tests/golden/gemm_f16x3_tail_shapes.npz

These fixtures show that nothing changed, not that the output is right; correctness is checked independently by
tests/test_gpu_gemm_probe.py (the kernel called directly, against float64 and bit-exact host models of every epilogue
mode) and tests/test_gpu_dense_lift_window.py (the fused leapfrog at rows that leave the planes' exact lift window).
"""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

import test_gpu_gemm_bit_identity as bit  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(HERE, "golden", "gemm_f16x3_tail_shapes.npz")
# (chains, dims, per-chain step sizes)
CASES = [(1, 1024, True), (70, 260, False), (129, 644, True)]


@pytest.mark.parametrize("C, D, per_chain_eps", CASES)
def test_tail_shape_products_bit_identical(C, D, per_chain_eps):
    want = np.load(GOLDEN)
    got = bit.case_outputs(C, D, per_chain_eps)
    for name, a in got.items():
        f, b = bit.fingerprint(a), want[bit._key(C, D, name)]
        assert f.shape == b.shape and f.dtype == b.dtype, name
        rows = np.flatnonzero(bit._bits(f) != bit._bits(b))
        assert rows.size == 0, f"{name}: rows {rows[:16].tolist()} ({rows.size} of {len(f)}) differ from the recorded bits"


if __name__ == "__main__":
    arrays = {}
    for C, D, per_chain_eps in CASES:
        arrays.update({bit._key(C, D, k): bit.fingerprint(v) for k, v in bit.case_outputs(C, D, per_chain_eps).items()})
    np.savez_compressed(sys.argv[1], **arrays)
    print(f"wrote {len(arrays)} arrays to {sys.argv[1]}")
