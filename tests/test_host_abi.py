"""CPU-only tests: the C-ABI library loads and exports every symbol include/bjx.h declares, argument
errors surface as they should without a GPU, and the host-side adaptation logic (schedule, shared-epsilon
dual averaging, CGL merge, the one all-gather under gloo with world_size 2) matches the oracle."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "bjx.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(bjx_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from blackjax_b200 import _lib
    lib = _lib.lib()
    declared = _declared_symbols()
    assert len(declared) >= 35
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/bjx.h but not exported by libbjx.so"
    assert sorted(_lib.EXPORTED_SYMBOLS) == declared      # the ctypes binding covers the whole header
    assert lib.bjx_version() == 100


def test_struct_layouts_match_header():
    from blackjax_b200 import _lib
    # bjx_target_desc: 2 x int32, 3 pointers, float (+pad), 2 pointers, 2 x int32, 2 pointers; bjx_info: 14 pointers
    assert C.sizeof(_lib.TargetDesc) == 80
    assert _lib.TargetDesc.user_params.offset == 64 and _lib.TargetDesc.user_plugin.offset == 72
    assert C.sizeof(_lib.Info) == 14 * 8
    assert C.sizeof(_lib.Config) == 16 + 8 + 8 + 80


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback_fails_loudly():
    import blackjax_b200 as bj
    from blackjax_b200 import _lib
    cfg = _lib.Config()
    cfg.device, cfg.n_chains, cfg.dim, cfg.max_tree_depth = 0, 4, 8, 10
    cfg.target.kind, cfg.target.dim = _lib.TARGET_FUNNEL, 8
    h = C.c_void_p()
    rc = _lib.lib().bjx_create(C.byref(cfg), C.byref(h))
    assert rc > 0                                          # a cudaError_t, not a silent CPU path
    assert b"no CPU fallback" in _lib.lib().bjx_last_error(None)
    with pytest.raises(TypeError, match="CUDA tensor"):
        bj.hmc.init(torch.zeros(4, 8), bj.targets.Funnel(8))


def test_argument_validation_without_gpu():
    from blackjax_b200 import _lib
    lib = _lib.lib()
    h = C.c_void_p()
    assert lib.bjx_create(None, C.byref(h)) == -1
    cfg = _lib.Config()
    cfg.device, cfg.n_chains, cfg.dim, cfg.max_tree_depth = 0, 0, 8, 10
    assert lib.bjx_create(C.byref(cfg), C.byref(h)) == -1
    cfg.n_chains, cfg.dim = 4, 1030                        # dim % 4 != 0 and > 128
    assert lib.bjx_create(C.byref(cfg), C.byref(h)) == -2
    assert lib.bjx_init_state(None, None, None, None) == -1


def test_api_surface_mirrors_blackjax():
    import inspect

    import blackjax_b200 as bj
    for alg in (bj.hmc, bj.nuts):
        assert callable(alg) and callable(alg.init) and callable(alg.build_kernel)
        assert list(inspect.signature(alg.init).parameters)[:2] == ["position", "logdensity_fn"]
    k = bj.hmc.build_kernel()
    assert list(inspect.signature(k).parameters) == ["rng_key", "state", "logdensity_fn", "step_size",
                                                     "inverse_mass_matrix", "num_integration_steps"]
    k = bj.nuts.build_kernel()
    assert list(inspect.signature(k).parameters)[:6] == ["rng_key", "state", "logdensity_fn", "step_size",
                                                         "inverse_mass_matrix", "max_num_doublings"]
    alg = bj.nuts(bj.targets.Funnel(8), 0.1, torch.ones(8))
    assert isinstance(alg, bj.SamplingAlgorithm)
    assert list(inspect.signature(alg.step).parameters) == ["rng_key", "state"]
    assert bj.nuts.init is bj.hmc.init                     # blackjax/mcmc/nuts.py:33
    # blackjax/__init__.py:117-118,154-162 and mcmc/dynamic_hmc.py:54-60,97-104
    assert bj.dynamic_hmc is bj.dhmc and callable(bj.dmhmc.build_kernel)
    assert list(inspect.signature(bj.dhmc.init).parameters) == ["position", "logdensity_fn", "random_generator_arg"]
    assert list(inspect.signature(bj.dhmc.build_kernel()).parameters) == [
        "rng_key", "state", "logdensity_fn", "step_size", "inverse_mass_matrix", "integration_steps_params"]
    assert bj.mcmc.dynamic_hmc.DynamicHMCState._fields == ("position", "logdensity", "logdensity_grad",
                                                           "random_generator_arg")


def test_schedule_matches_reference_kat():
    import blackjax_b200 as bj
    from oracle.adaptation import build_schedule as ob
    for n in (0, 5, 19, 20, 37, 100, 150, 200, 1000):
        assert bj.build_schedule(n) == ob(n)
    assert bj.build_schedule(100) == [(0, False)] * 15 + [(1, False)] * 74 + [(1, True)] + [(0, False)] * 10


def test_shared_dual_averaging_host_matches_oracle():
    import importlib
    wa = importlib.import_module("blackjax_b200.adaptation.window_adaptation")
    from oracle import adaptation as oa
    rs = np.random.default_rng(0)
    s, o = wa._da_init(0.7), oa.da_init(0.7)
    for _ in range(40):
        a = float(rs.uniform(0, 1))
        s, o = wa._da_update(s, a, 0.8), oa.da_update(o, a, 0.8)
        assert s.log_step == pytest.approx(float(o.log_step_size), rel=1e-6, abs=1e-7)
        assert s.log_step_avg == pytest.approx(float(o.log_step_size_avg), rel=1e-6, abs=1e-7)
        assert s.step == o.step


def test_cgl_merge_blocks_matches_oracle():
    from blackjax_b200.adaptation.window_adaptation import cgl_merge_blocks
    from oracle import adaptation as oa
    rs = np.random.default_rng(1)
    D, G = 7, 4
    xs = [rs.standard_normal((50 + 10 * g, D)).astype(np.float32) * (g + 1) for g in range(G)]
    blocks = []
    for x in xs:
        m = x.mean(0)
        blocks.append(np.concatenate([[x[:, 0].sum()], [len(x)], m, ((x - m) ** 2).sum(0)]))
    acc, n, mean, m2 = cgl_merge_blocks(torch.tensor(np.stack(blocks), dtype=torch.float32))
    allx = np.concatenate(xs)
    assert float(n) == len(allx)
    np.testing.assert_allclose(mean.numpy(), allx.mean(0), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(m2.numpy(), ((allx - allx.mean(0)) ** 2).sum(0), rtol=1e-4)
    w = oa.Welford(blocks[0][2:2 + D].astype(np.float32), blocks[0][2 + D:].astype(np.float32), len(xs[0]))
    for b, x in zip(blocks[1:], xs[1:]):
        w = oa.cgl_merge(w, oa.Welford(b[2:2 + D].astype(np.float32), b[2 + D:].astype(np.float32), len(x)))
    np.testing.assert_allclose(m2.numpy(), w.m2, rtol=1e-5)


def test_cgl_merge_blocks_dense_matches_numpy():
    from blackjax_b200.adaptation.window_adaptation import cgl_merge_blocks
    rs = np.random.default_rng(2)
    D, G = 5, 3
    xs = [rs.standard_normal((40 + 7 * g, D)) @ rs.standard_normal((D, D)) for g in range(G)]
    blocks = []
    for x in xs:
        m = x.mean(0)
        blocks.append(np.concatenate([[1.0], [len(x)], m, ((x - m).T @ (x - m)).ravel()]))
    acc, n, mean, m2 = cgl_merge_blocks(torch.tensor(np.stack(blocks), dtype=torch.float32), D)
    allx = np.concatenate(xs)
    assert m2.shape == (D, D) and float(n) == len(allx)
    np.testing.assert_allclose(m2.numpy(), (allx - allx.mean(0)).T @ (allx - allx.mean(0)), rtol=1e-4, atol=1e-3)


_GLOO_WORKER = r"""
import os, sys, numpy as np, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from blackjax_b200.adaptation.window_adaptation import _allgather_stats, cgl_merge_blocks
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:" + sys.argv[2], rank=int(sys.argv[3]), world_size=2)
rank = dist.get_rank()
rs = np.random.default_rng(0)
D = 5
x_all = rs.standard_normal((64, D)).astype(np.float32) * 2 + 1
acc_all = rs.uniform(0, 1, 64).astype(np.float32)
x, a = x_all[rank * 32:(rank + 1) * 32], acc_all[rank * 32:(rank + 1) * 32]        # chain shard of this rank
m = x.mean(0)
block = torch.tensor(np.concatenate([[a.sum()], [32.0], m, ((x - m) ** 2).sum(0)]), dtype=torch.float32)
blocks = _allgather_stats(block, None)                                            # the ONE collective
acc, n, mean, m2 = cgl_merge_blocks(blocks)
assert blocks.shape == (2, 2 + 2 * D) and float(n) == 64
np.testing.assert_allclose(float(acc) / float(n), acc_all.mean(), rtol=1e-5)
np.testing.assert_allclose(mean.numpy(), x_all.mean(0), rtol=1e-5, atol=1e-6)
np.testing.assert_allclose(m2.numpy(), ((x_all - x_all.mean(0)) ** 2).sum(0), rtol=1e-4)
# every rank must hold bit-identical merged statistics (no broadcast follows)
gathered = [torch.empty_like(m2) for _ in range(2)]
dist.all_gather(gathered, m2)
assert torch.equal(gathered[0], gathered[1])
# dense mass-matrix adaptation: the block carries the full [D, D] matrix of co-moments (bjx_pooled_stats_dense layout)
xc = x - m
blockd = torch.tensor(np.concatenate([[a.sum()], [32.0], m, (xc.T @ xc).ravel()]), dtype=torch.float32)
blocksd = _allgather_stats(blockd, None)
accd, nd, meand, m2d = cgl_merge_blocks(blocksd, dim=D)
assert blocksd.shape == (2, 2 + D + D * D) and m2d.shape == (D, D) and float(nd) == 64
xa = x_all - x_all.mean(0)
np.testing.assert_allclose(m2d.numpy(), xa.T @ xa, rtol=1e-4, atol=1e-3)
np.testing.assert_allclose(meand.numpy(), x_all.mean(0), rtol=1e-5, atol=1e-6)
gathered = [torch.empty_like(m2d) for _ in range(2)]
dist.all_gather(gathered, m2d)
assert torch.equal(gathered[0], gathered[1])
dist.destroy_process_group()
print("OK", rank)
"""


def test_allgather_merge_world_size_2_gloo(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(_GLOO_WORKER)
    port = str(29500 + (os.getpid() % 2000))
    procs = [subprocess.Popen([sys.executable, str(script), ROOT, port, str(r)], stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT) for r in range(2)]
    outs = [p.communicate(timeout=180)[0].decode() for p in procs]
    for p, o in zip(procs, outs):
        assert p.returncode == 0, o
        assert "OK" in o


@pytest.mark.parametrize("workload", ["hmc_iso_gaussian_1024x100_L10", "hmc_hier_logit_32768x10000_L20"])
def test_bench_reference_arm_contract(workload):
    """`bench.py --impl reference` (the CPU arm the driver times beside ours) runs without a GPU, prints exactly one
    JSON line on stdout and carries the contract's keys; the product arm refuses to run without a GPU."""
    import json
    import subprocess
    import sys
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--workload",
           workload, "--steps", "2", "--warmup", "1"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "leapfrog-steps/s" and d["higher_is_better"] is True
    assert d["value"] > 0 and d["steps"] == 2 and d["warmup"] == 1 and d["n_gpus"] == 1
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert d["config"]["workload"] == workload
    if not torch.cuda.is_available() and workload.startswith("hmc_iso"):
        ours = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "1", "--warmup", "1"],
                              capture_output=True, text=True, timeout=300, cwd=ROOT)
        assert ours.returncode != 0          # no silent CPU path


def test_library_is_sm90a_with_wgmma_and_tma_sass():
    """Static evidence that the shipped library is Hopper code, not a recompiled generic kernel: every cubin is
    sm_90a, and the dense path's GEMM issues asynchronous warpgroup MMAs (HGMMA) on operands that TMA (UTMALDG) lands
    in shared memory behind mbarriers (SYNCS)."""
    import shutil
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    so = os.path.join(ROOT, "blackjax_b200", "libbjx.so")
    sass = subprocess.run([cuobjdump, "-sass", so], capture_output=True, text=True, timeout=600).stdout
    archs = {l.split("=")[1].strip() for l in sass.splitlines() if l.startswith("arch =")}
    assert archs == {"sm_90a"}, archs
    for mnemonic in ("HGMMA.64x128x16.F32", "UTMALDG", "SYNCS"):
        assert mnemonic in sass, f"{mnemonic} missing from libbjx.so SASS"
    assert "HMMA.16816" not in sass      # no mma.sync fallback


def test_dense_gaussian_rejects_an_asymmetric_precision():
    """The fused value_and_grad computes -P x, the gradient of -1/2 x^T P x only for symmetric P (ADVICE round 1)."""
    import numpy as np
    import pytest
    from blackjax_b200 import targets as T
    P = np.eye(4) + 0.1 * np.triu(np.ones((4, 4)), 1)
    with pytest.raises(ValueError, match="symmetric"):
        T.DenseGaussian(P)
    T.DenseGaussian(0.5 * (P + P.T))


# ---- user-defined target plug-ins (include/bjx_user_target.h): host-side machinery, no compute ---------------------
def test_plugin_builds_exports_and_loads():
    from blackjax_b200 import _lib, plugin
    path = plugin.build_plugin(plugin.read_example("diag_gaussian"), 18, "diag_gaussian", dense_metric=False,
                               general_integrators=False)
    assert path.startswith(plugin.PLUGIN_DIR) and os.path.exists(path)
    so = C.CDLL(path)
    assert so.bjx_plugin_built_for_abi() == _lib.lib().bjx_plugin_abi()
    assert hasattr(so, "bjx_plugin_launch")
    p = plugin.load_plugin(path)
    assert p and plugin.load_plugin(path) == p            # cached per path
    # same source, another row size class or other options: another build
    other, _ = plugin.plugin_path(plugin.read_example("diag_gaussian"), 100, "diag_gaussian", False, False)
    assert other != path
    same, _ = plugin.plugin_path(plugin.read_example("diag_gaussian"), 21, "diag_gaussian", False, False)
    assert same == path                                    # 18 and 21 dims share the scalar <= 32 size class


def test_big_row_plugin_builds_and_exports_its_launcher():
    # rows beyond a warp: the CTA-level contract (bjx_user::BigModel); the plug-in exports bjx_plugin_launch_big only
    from blackjax_b200 import _lib, plugin
    assert plugin.size_class(2048) == plugin.SC_BIG and plugin.size_class(18432) == plugin.SC_BIG
    path = plugin.build_plugin(plugin.read_example("diag_gaussian_big"), 2048, "diag_gaussian_big", False, False)
    so = C.CDLL(path)
    assert so.bjx_plugin_built_for_abi() == _lib.lib().bjx_plugin_abi()
    assert hasattr(so, "bjx_plugin_launch_big") and not hasattr(so, "bjx_plugin_launch")
    assert plugin.load_plugin(path)
    # the options of the warp kernels do not apply to this size class: one build whatever they say
    assert plugin.plugin_path(plugin.read_example("diag_gaussian_big"), 4096, "diag_gaussian_big", True, True)[0] == path


def test_plugin_load_rejects_foreign_libraries_and_missing_files():
    from blackjax_b200 import _lib
    out = C.c_void_p()
    assert _lib.lib().bjx_plugin_load(b"/nonexistent/libbjxt.so", C.byref(out)) == -1
    assert b"bjx_plugin_load" in _lib.lib().bjx_last_error(None)
    assert _lib.lib().bjx_plugin_load(_lib.LIB_PATH.encode(), C.byref(out)) == -1     # libbjx itself is not a plug-in
    assert b"not a bjx target plug-in" in _lib.lib().bjx_last_error(None)


def test_plugin_compile_error_is_reported_with_the_compiler_output():
    from blackjax_b200 import BjxError, plugin
    bad = "namespace bjx_user { template <class R> struct Model { this is not CUDA }; }"
    with pytest.raises(BjxError, match="nvcc failed"):
        plugin.build_plugin(bad, 8, "broken", dense_metric=False, general_integrators=False)
    path, _ = plugin.plugin_path(bad, 8, "broken", False, False)
    assert not os.path.exists(path)


def test_plugin_size_classes_mirror_the_launcher():
    from blackjax_b200 import plugin
    assert [plugin.size_class(d) for d in (4, 128, 132, 256, 260, 512, 516, 1024, 1, 31, 33, 127)] == \
        [0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5]
    for d in (0, 130, 1030, 18436):
        with pytest.raises(ValueError):
            plugin.size_class(d)


def test_user_target_descriptor_without_gpu():
    # building the descriptor loads the plug-in and needs the parameter block on a device: without a GPU the
    # constructor and the build still work, and the linear regression packs [N, K, X, y]
    from blackjax_b200 import targets
    x = np.arange(12, dtype=np.float32).reshape(4, 3)
    y = np.ones(4, np.float32)
    t = targets.LinearRegression(x, y, dense_metric=False, general_integrators=False)
    assert t.dim == 4 and t.params.shape == (2 + 12 + 4,) and t.params[0] == 4 and t.params[1] == 3
    assert os.path.exists(t.plugin_path())
    with pytest.raises(ValueError):
        targets.LinearRegression(np.zeros((4, 17), np.float32), y)


def test_headers_are_valid_c99(tmp_path):
    """include/bjx.h is the drop-in boundary for non-C++ hosts (cgo, JNI, ctypes generators): it must compile as plain C."""
    src = tmp_path / "abi.c"
    src.write_text('#include "bjx.h"\n#include "bjx_user_target.h"\n'
                   'int probe(void) { bjx_config c; bjx_info i; bjx_target_desc t; (void)c; (void)i; (void)t;\n'
                   '  return (int)sizeof(bjx_handle_t) + BJX_TARGET_USER + BJX_METRIC_DENSE_PER_CHAIN + BJX_E_STATE; }\n')
    inc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include")
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", inc, "-c", str(src), "-o",
                        str(tmp_path / "abi.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_plugin_cubins_are_sm90a_with_the_same_kernels_as_the_library():
    """A user-defined target's plug-in holds the path's kernels compiled for sm_90a only -- the same templates as the
    built-in row kernels, another translation unit."""
    import shutil
    from blackjax_b200 import plugin
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    path = plugin.build_plugin(plugin.read_example("diag_gaussian"), 256, "diag_gaussian", dense_metric=False,
                               general_integrators=False)
    elf = subprocess.run([cuobjdump, "-lelf", path], capture_output=True, text=True, timeout=120).stdout
    archs = set(re.findall(r"sm_\d+a?", elf))
    assert archs == {"sm_90a"}, archs
    sass = subprocess.run([cuobjdump, "-sass", path], capture_output=True, text=True, timeout=600).stdout
    for kern in ("k_hmc_transition", "k_mhmc_transition", "k_ghmc_transition", "k_nuts_doubling", "k_nuts_chains", "k_leapfrog",
                 "k_init_state"):
        assert kern in sass, kern
    assert re.search(r"k_hmc_transitionINS_3RowILi8ELb1EEELi4E", sass), "HMC kernel of the user target (Row<8,true>, TK=4) missing"
