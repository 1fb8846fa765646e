"""The sm_90a compile of the dense path's tensor-core product (bjx::k_gemm_f16x3, bjx_gemm.cu), read from ptxas -v.

The kernel keeps two accumulator sets per consumer thread and a tile's epilogue inputs in registers; a spill would put
local-memory traffic into the K loop.  ptxas also serializes wgmma.mma_async on its own, with only an advisory, when it
cannot prove that the accumulators are left alone between a wgmma's issue and the wait that completes it; the kernel
then still computes the same sums, but its MMAs no longer overlap its epilogue.  No GPU is needed, only nvcc."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "blackjax_b200", "csrc")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CLEAN = " 0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads"


def makefile_flags():
    """NVFLAGS of blackjax_b200/csrc/Makefile with $(ARCH) expanded."""
    text = open(os.path.join(CSRC, "Makefile")).read()
    arch = re.search(r"^ARCH\s*:=\s*(.*)$", text, re.M).group(1).split()
    flags = re.search(r"^NVFLAGS\s*:=\s*(.*)$", text, re.M).group(1).split()
    return [a for f in flags for a in (arch if f == "$(ARCH)" else [f])]


@pytest.mark.skipif(not os.path.exists(NVCC), reason="needs nvcc")
def test_gemm_compiles_without_spills_or_serialized_wgmma(tmp_path):
    out = subprocess.run([NVCC, *makefile_flags(), "-Xptxas", "-v", "-c", os.path.join(CSRC, "bjx_gemm.cu"), "-o",
                          str(tmp_path / "bjx_gemm.o")], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-2000:]
    log = out.stderr
    assert "sm_90a" in log, log
    assert "wgmma.mma_async instructions are serialized" not in log, log
    blocks = [b for b in log.split("Compiling entry function")[1:] if "k_gemm_f16x3" in b.split("\n")[0]]
    assert len(blocks) == 1, log
    assert CLEAN in blocks[0], blocks[0]
