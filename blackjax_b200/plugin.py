"""Build and load plug-ins of user-defined targets (include/bjx_user_target.h).

The reference differentiates any ``logdensity_fn`` callable with ``jax.value_and_grad`` (blackjax/mcmc/hmc.py:91,
integrators.py:189); its "compiler" is XLA.  Here the user supplies the fused ``value_and_grad`` as CUDA source and this
module runs nvcc on ``csrc/bjx_plugin.cu`` + that source: one shared library per (source, row size class, options),
cached IN-TREE under ``blackjax_b200/_plugins/`` (so a prebuilt plug-in travels with the package like libbjx.so itself).
There is no interpreter fallback: without nvcc and without a cached build the target cannot be created.
"""
import ctypes as C
import hashlib
import os
import shutil
import subprocess

from . import _lib

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
INCLUDE = os.path.join(os.path.dirname(_HERE), "include")
PLUGIN_DIR = os.path.join(_HERE, "_plugins")
USER_TARGETS = os.path.join(_HERE, "user_targets")

# everything a plug-in is compiled from besides the user's source: a change in any of these is a new build
_ABI_SOURCES = ("bjx_plugin.cu", "bjx_row.cuh", "bjx_kernels.cuh", "bjx_launch.cuh", "bjx_prng.cuh", "bjx_big.cuh")

SC_BIG = 6
_LOADED = {}  # path -> bjx_plugin pointer (plug-ins stay loaded for the life of the process)


def size_class(dim):
    """Row size class of the kernels (csrc/bjx_launch.cuh ``size_class_for``): 0..5 the warp kernels (rows up to 1024 dims,
    the model is a ``bjx_user::Model<R>``), 6 the CTA-per-chain kernels (1024 < dim <= 18432, ``bjx_user::BigModel``)."""
    if dim <= 0:
        raise ValueError("dim must be positive")
    if dim % 4 == 0 and dim <= 1024:
        return 0 if dim <= 128 else 1 if dim <= 256 else 2 if dim <= 512 else 3
    if dim <= 32:
        return 4
    if dim <= 128:
        return 5
    if dim % 4 == 0 and dim <= 18432:
        return SC_BIG
    raise ValueError("user-defined targets need dim <= 18432 with dim % 4 == 0, or dim <= 128 otherwise")


def _nvcc():
    for cand in (os.environ.get("BJX_NVCC"), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc"),
                 shutil.which("nvcc")):
        if cand and os.path.exists(cand):
            return cand
    return None


def _abi_digest():
    h = hashlib.sha256()
    for name in _ABI_SOURCES:
        with open(os.path.join(CSRC, name), "rb") as f:
            h.update(f.read())
    with open(os.path.join(INCLUDE, "bjx.h"), "rb") as f:
        h.update(f.read())
    return h


def plugin_path(source, dim, name="user", dense_metric=True, general_integrators=True):
    """Where the plug-in of this (source text, row size class, options) lives, whether or not it has been built."""
    h = _abi_digest()
    sc = size_class(dim)
    flags = (sc, 2 if dense_metric else 0, 2 if general_integrators else 0)
    if sc == SC_BIG:  # diagonal metrics and velocity Verlet only in this size class: the options do not apply
        flags = (sc, 0, 0)
    h.update(repr(flags).encode())
    h.update(source.encode())
    safe = "".join(ch if ch.isalnum() else "_" for ch in name)[:40]
    return os.path.join(PLUGIN_DIR, f"libbjxt_{safe}_{h.hexdigest()[:16]}.so"), flags


def build_plugin(source, dim, name="user", dense_metric=True, general_integrators=True, verbose=False):
    """Compile (once) the plug-in for ``source`` -- CUDA text defining ``bjx_user::Model`` -- at this row size.

    ``dense_metric`` / ``general_integrators``: also build the small-dense / low-rank metric variants and the
    mclachlan / yoshida / omelyan integrator variants (each doubles the compile time: about 8 s without both, 30 s with
    both, per row size class).  Returns the path of the shared library."""
    path, (sc, dm, gen) = plugin_path(source, dim, name, dense_metric, general_integrators)
    if os.path.exists(path):
        return path
    nvcc = _nvcc()
    if nvcc is None:
        raise _lib.BjxError(f"cannot build the target plug-in {os.path.basename(path)}: nvcc not found (set CUDA_HOME or "
                            "BJX_NVCC); user-defined targets have no interpreted fallback")
    os.makedirs(PLUGIN_DIR, exist_ok=True)
    src = path[:-3] + ".cuh"
    with open(src, "w") as f:
        f.write(source)
    tmp = path + f".tmp{os.getpid()}"
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
           "-shared", "-I", CSRC, "-I", INCLUDE, f"-DBJX_USER_SOURCE=\"{src}\""]
    if sc == SC_BIG:
        cmd += ["-DBJX_PLUGIN_BIG=1"]
    else:
        cmd += [f"-DBJX_BUILD_SC={sc}", f"-DBJX_BUILD_DM={dm}", f"-DBJX_BUILD_GEN={gen}"]
    cmd += [os.path.join(CSRC, "bjx_plugin.cu"), "-o", tmp]
    if verbose:
        print(" ".join(cmd))
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        if os.path.exists(tmp):
            os.remove(tmp)
        raise _lib.BjxError(f"nvcc failed on the user-defined target '{name}':\n{r.stdout}\n{r.stderr}")
    os.replace(tmp, path)  # atomic: concurrent ranks may build the same plug-in
    return path


def load_plugin(path):
    """bjx_plugin_load (include/bjx.h): open the library, check it was built against this libbjx, return the pointer."""
    p = _LOADED.get(path)
    if p is None:
        out = C.c_void_p()
        _lib.check(_lib.lib().bjx_plugin_load(path.encode(), C.byref(out)))
        p = _LOADED[path] = out.value
    return p


def read_example(name):
    """Source text of a target shipped in blackjax_b200/user_targets/ (e.g. 'linear_regression')."""
    with open(os.path.join(USER_TARGETS, name + ".cuh")) as f:
        return f.read()


# Plug-ins the test-suite and smoke() use, prebuilt by __graft_entry__.build() so they travel with the snapshot:
# (example, dim, dense_metric, general_integrators)
PREBUILT = (
    ("diag_gaussian", 100, True, True),     # SC_V1
    ("diag_gaussian", 18, False, False),    # SC_S1
    ("diag_gaussian", 70, False, False),    # SC_S4
    ("diag_gaussian", 256, False, False),   # SC_V2
    ("diag_gaussian", 512, False, False),   # SC_V4
    ("diag_gaussian", 1024, False, False),  # SC_V8
    ("linear_regression", 2, True, True),   # SC_S1: the reference's regression posterior (log_scale + K <= 16 coefficients)
    ("linear_regression", 4, True, True),   # SC_V1 (three or seven coefficients: 4 or 8 dims)
    ("rosenbrock", 5, False, False), ("rosenbrock", 100, False, False), ("rosenbrock", 70, False, False),
    ("rosenbrock", 256, False, False), ("rosenbrock", 1024, False, False),   # SC_S1, V1, S4, V2, V8
    ("diag_gaussian_big", 2048, False, False), ("hier_logit_big", 1504, False, False),   # CTA-per-chain rows (SC_BIG)
    ("bounded_gaussian", 2, False, True),   # SC_S1: MCLMC's NaN handling (a box whose overshoots give NaN log-densities)
)


def build_prebuilt(verbose=False):
    from concurrent.futures import ThreadPoolExecutor
    jobs = [(read_example(ex), dim, ex, dm, gen) for ex, dim, dm, gen in PREBUILT]
    with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 1)) as pool:
        return list(pool.map(lambda j: build_plugin(*j, verbose=verbose), jobs))
