"""The sm_90a compile of the fused kernels, read from ptxas -v: no stack frame and no local-memory spills.

Each case compiles one translation unit with its own nvcc flags: the MCLMC, adjusted MCLMC and MCLMC tuning kernels
instantiated over every row size class and both integrator forms, the MEADS-LRD eigensolver kernels of bjx_meads.cu and
the low-rank window adaptation kernels of bjx_lowrank_window.cu.  No GPU is needed, only nvcc."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "blackjax_b200", "csrc")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CLEAN = " 0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads"

# every row size class with the diagonal Gaussian, plus the other built-in targets at the size classes they run on
INSTANCES = [(r, "TK_DIAG") for r in ("Row<1, false>", "Row<4, false>", "Row<4, true>", "Row<8, true>", "Row<16, true>",
                                      "Row<32, true>")] + [("Row<32, true>", "TK_FUNNEL"), ("Row<4, true>", "TK_DENSE"),
                                                           ("Row<1, false>", "TK_BANANA")]
MCLMC_TRANSITION = ("k_mclmc_transition", "Params, const uint32_t*, float*, float*, float*, float*, MclmcArgs")
AMCLMC_TRANSITION = ("k_amclmc_transition", "Params, const uint32_t*, const float*, const float*, const float*, float*, "
                                            "float*, float*, AmclmcArgs, InfoPtrs")
MCLMC_TUNE = ("k_mclmc_tune", "Params, const uint32_t*, float*, float*, float*, float*, MclmcTuneArgs")
WITH_CSRC = ["-Xptxas", "-v", "-I", CSRC]


def instantiate(*kernels):
    """A translation unit that instantiates each (kernel, parameter list) for every instance and both integrator forms
    (the velocity Verlet specialisation and the general coefficient table)."""
    lines = ['#include "bjx_kernels.cuh"', "namespace bjx {"]
    for row, tk in INSTANCES:
        for gen in ("false", "true"):
            for name, params in kernels:
                lines.append(f"template __global__ void {name}<{row}, {tk}, false, {gen}>({params});")
    return "\n".join(lines + ["}"]) + "\n"


def ptxas_log(tmp_path, source, flags):
    """ptxas' report of nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 <flags> -c on source, a file of the
    repository or the text of a translation unit."""
    if not os.path.isfile(source):
        (tmp_path / "inst.cu").write_text(source)
        source = str(tmp_path / "inst.cu")
    out = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", *flags, "-c", source,
                          "-o", str(tmp_path / "k.o")], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-2000:]
    return out.stderr


def assert_entries_clean(log, names, count):
    """Exactly count entry functions whose names contain one of names, each without stack frame or spills."""
    blocks = [b for b in re.split(r"Compiling entry function", log) if any(n in b.split("\n")[0] for n in names)]
    assert len(blocks) == count, [b.split("\n")[0] for b in blocks]
    for b in blocks:
        assert CLEAN in b, b


CASES = {  # (translation unit, nvcc flags, entry names, entries expected: None checks every function of the unit)
    "k_mclmc_transition": (instantiate(MCLMC_TRANSITION), WITH_CSRC, ("k_mclmc_transition",), 2 * len(INSTANCES)),
    "k_amclmc_transition": (instantiate(AMCLMC_TRANSITION), WITH_CSRC, ("k_amclmc_transition",), 2 * len(INSTANCES)),
    "k_mclmc_tune": (instantiate(MCLMC_TUNE), WITH_CSRC, ("k_mclmc_tune",), 2 * len(INSTANCES)),
    "k_lrd": (os.path.join(CSRC, "bjx_meads.cu"), ["-Xcompiler", "-fPIC", "-Xptxas", "-v"], ("k_lrd_",), 4),
    "bjx_lowrank_window": (os.path.join(CSRC, "bjx_lowrank_window.cu"),
                           ["-Xptxas", "-v", "-I", os.path.join(ROOT, "include")], ("k_lw_final", "k_lw_merge"), None),
}


@pytest.mark.skipif(not os.path.exists(NVCC), reason="needs nvcc")
@pytest.mark.parametrize("case", list(CASES))
def test_kernels_compile_without_spills(case, tmp_path):
    source, flags, names, count = CASES[case]
    log = ptxas_log(tmp_path, source, flags)
    if count is not None:
        assert_entries_clean(log, names, count)
    else:  # the named entries are there, and every function ptxas reports on is clean
        assert all(n in log for n in names), names
        reports = [ln for ln in log.splitlines() if "spill" in ln]
        assert reports and all(CLEAN in ln for ln in reports), reports
