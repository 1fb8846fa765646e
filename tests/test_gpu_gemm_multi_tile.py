"""Bit-identity of the dense path's tensor-core product (bjx::k_gemm_f16x3, bjx_gemm.cu) at shapes with more tiles than
CTAs, where every CTA runs two or more tiles and a tile's epilogue runs under the next tile's K loop:

  (4500, 1024, True)   288 tiles: 8 column tiles per row block, a 20-row tail, 16 K blocks;
  (9000, 644, False)   426 tiles: 6 column tiles, the last one 4 columns wide, 11 K blocks, the last one 4 deep;
  (20000, 200, True)   314 tiles: 2 column tiles, 4 K blocks (fewer K blocks than epilogue slices).

tests/test_gpu_gemm_bit_identity.py and tests/test_gpu_gemm_tail_shapes.py run at most 16 tiles, one per CTA.
Products and inputs are those of tests/test_gpu_gemm_bit_identity.py, imported from it.  To keep the fixture small,
the per-row fingerprints of that file (a row digest, or a log-density as it is) are digested once more per block of
128 rows, one row tile of the product; a changed bit changes its block's digest, and the failure names the blocks.

The fixture tests/golden/gemm_f16x3_multi_tile.npz holds the outputs of the kernel of commit 0a0c28c, whose epilogue ran
after its tile's K loop, recorded on an H100 80GB HBM3 by running this file with the library built from that commit:
    python tests/test_gpu_gemm_multi_tile.py tests/golden/gemm_f16x3_multi_tile.npz

These fixtures show that nothing changed, not that the output is right; correctness is checked independently by
tests/test_gpu_gemm_probe.py (the kernel called directly, against float64 and bit-exact host models of every epilogue
mode) and tests/test_gpu_dense_lift_window.py (the fused leapfrog at rows that leave the planes' exact lift window).
"""
import hashlib
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

import test_gpu_gemm_bit_identity as bit  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(HERE, "golden", "gemm_f16x3_multi_tile.npz")
# (chains, dims, per-chain step sizes)
CASES = [(4500, 1024, True), (9000, 644, False), (20000, 200, True)]
BLOCK = 128


def block_fingerprint(a):
    """One 64-bit BLAKE2b digest of the row fingerprints of every block of BLOCK rows."""
    rows = np.ascontiguousarray(bit.fingerprint(a))
    return np.array([int.from_bytes(hashlib.blake2b(rows[i:i + BLOCK].tobytes(), digest_size=8).digest(), "little")
                     for i in range(0, len(rows), BLOCK)], np.uint64)


@pytest.mark.parametrize("C, D, per_chain_eps", CASES)
def test_multi_tile_products_bit_identical(C, D, per_chain_eps):
    want = np.load(GOLDEN)
    got = bit.case_outputs(C, D, per_chain_eps)
    for name, a in got.items():
        f, b = block_fingerprint(a), want[bit._key(C, D, name)]
        assert f.shape == b.shape and f.dtype == b.dtype, name
        blocks = np.flatnonzero(f != b)
        assert blocks.size == 0, (f"{name}: rows {[(BLOCK * i, BLOCK * (i + 1)) for i in blocks[:8]]} ({blocks.size} of "
                                  f"{len(f)} blocks of {BLOCK} rows) differ from the recorded bits")


if __name__ == "__main__":
    arrays = {}
    for C, D, per_chain_eps in CASES:
        arrays.update({bit._key(C, D, k): block_fingerprint(v) for k, v in bit.case_outputs(C, D, per_chain_eps).items()})
    np.savez_compressed(sys.argv[1], **arrays)
    print(f"wrote {len(arrays)} arrays to {sys.argv[1]}")
