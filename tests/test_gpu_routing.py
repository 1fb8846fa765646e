"""Which execution path every transition entry point of the C ABI takes, pinned by return code.

A handle runs on one of three paths: the warp-per-chain row kernels (dim <= 1024), the CTA-per-chain big-row kernels
(1024 < dim), or the tensor-core dense path (a dense metric or a dense Gaussian target beyond 128 dims).  Each path
rejects what it does not build: the general integrator and per-chain integration steps beyond the row kernels,
multinomial / generalized HMC, NUTS and the U-turn test on big rows, per-chain dense and low-rank metrics beyond their
dims, a plug-in without the kernels of the row size.  This test creates handles over a grid of target x dim x metric x
integrator that reaches every route and compares the return code of every entry point with tests/golden/routing_codes.json.
The codes only say which calls are accepted; the numbers the calls produce are checked by the parity tests, those of the
row kernels in every row size class (bjx_is_turning included) by tests/test_gpu_row_classes.py.
"""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from blackjax_b200 import _lib, plugin

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
N_CHAINS = 256
DIMS = (64, 256, 1028, 2048)
TARGETS = ("diag", "funnel", "dense", "hier_logit", "user_diag_gaussian", "user_diag_gaussian_big")
METRICS = ("diag", "dense", "diag_per_chain", "dense_per_chain", "low_rank")
INTEGRATORS = {"velocity_verlet": (0.5, 1.0, 0.5),
               "mclachlan": (0.1931833275037836, 0.5, 0.6136333449924328, 0.5, 0.1931833275037836)}
# the prebuilt plug-ins (plugin.PREBUILT), loaded at every dim: (source, row size it was built for)
PLUGINS = {"user_diag_gaussian": ("diag_gaussian", 256), "user_diag_gaussian_big": ("diag_gaussian_big", 2048)}
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "routing_codes.json")


class _Dev:
    """Device copies of numpy arrays, kept alive for the life of the handle that reads them."""

    def __init__(self):
        self.keep = []

    def __call__(self, a, dtype=np.float32):
        t = torch.from_numpy(np.ascontiguousarray(a, dtype)).to(DEV)
        self.keep.append(t)
        return t.data_ptr()


def _target(name, D, dev, rs):
    t = _lib.TargetDesc()
    t.dim = D
    if name == "diag":
        t.kind, t.inv_var = _lib.TARGET_DIAG_GAUSSIAN, dev(np.ones(D))
    elif name == "funnel":
        t.kind = _lib.TARGET_FUNNEL
    elif name == "dense":
        t.kind, t.precision = _lib.TARGET_DENSE_GAUSSIAN, dev(np.eye(D))
    elif name == "hier_logit":  # dim = 4 + n_groups; 8 observations of 2 covariates per group
        t.kind, t.n_groups = _lib.TARGET_HIER_LOGIT, D - 4
        t.data_x = dev(rs.standard_normal((D - 4, 16)))
        t.data_y = dev(rs.integers(0, 256, D - 4), np.int32)
    else:
        source, built_dim = PLUGINS[name]
        path = plugin.build_plugin(plugin.read_example(source), built_dim, source, dense_metric=False,
                                   general_integrators=False)
        t.kind, t.user_plugin = _lib.TARGET_USER, plugin.load_plugin(path)
        t.user_params, t.n_user_params = dev(np.ones(D)), D
    return t


def _set_metric(lib, h, metric, D, dev):
    if metric == "low_rank":
        rank = 2
        U = np.linalg.qr(np.random.default_rng(1).standard_normal((D, rank)))[0]
        return lib.bjx_set_metric_low_rank(h, dev(np.ones(D)), dev(U), dev(np.full(rank, 2.0)), rank)
    if metric == "diag":
        return lib.bjx_set_metric(h, _lib.METRIC_DIAG, dev(np.ones(D)))
    if metric == "dense":
        return lib.bjx_set_metric(h, _lib.METRIC_DENSE, dev(np.eye(D)))
    if metric == "diag_per_chain":
        return lib.bjx_set_metric(h, _lib.METRIC_DIAG_PER_CHAIN, dev(np.ones((N_CHAINS, D))))
    # per-chain dense metrics are refused beyond 64 dims before the matrices are read: no [C, D, D] array there
    imm = np.broadcast_to(np.eye(D), (N_CHAINS, D, D)) if D <= 64 else np.ones(1)
    return lib.bjx_set_metric(h, _lib.METRIC_DENSE_PER_CHAIN, dev(imm))


def _transition_codes(lib, h, D, metric, dev, rs):
    """Return code of every entry point, in a fixed order, on one handle (metric and integrator already set)."""
    Cn = N_CHAINS
    q, p, g = (dev(0.1 * rs.standard_normal((Cn, D))) for _ in range(3))
    logp, energy, slice_ = dev(np.zeros(Cn)), dev(np.zeros(Cn)), dev(np.zeros(Cn))
    turning = dev(np.zeros(Cn), np.uint8)
    keys = dev(rs.integers(0, 2**31, (Cn, 2)), np.int32)
    rng_key = dev(np.array([0, 42]), np.int32)
    steps = dev(np.full(Cn, 2), np.int32)
    eps = 0.01
    codes = {}
    codes["init_state"] = lib.bjx_init_state(h, q, logp, g)
    codes["sample_momentum"] = lib.bjx_sample_momentum(h, keys, p)
    codes["energy"] = lib.bjx_energy(h, p, logp, energy)
    codes["is_turning"] = lib.bjx_is_turning(h, p, p, p, turning)
    codes["leapfrog"] = lib.bjx_leapfrog(h, q, p, logp, g, eps, None, 2)
    codes["hmc_step"] = lib.bjx_hmc_step(h, keys, q, logp, g, q, logp, g, eps, None, 2, None)
    lib.bjx_set_integration_steps(h, steps)
    codes["hmc_step_per_chain_steps"] = lib.bjx_hmc_step(h, keys, q, logp, g, q, logp, g, eps, None, 2, None)
    lib.bjx_set_integration_steps(h, None)
    codes["mhmc_step"] = lib.bjx_mhmc_step(h, keys, q, logp, g, q, logp, g, eps, None, 2, None)
    codes["ghmc_step"] = lib.bjx_ghmc_step(h, keys, q, p, logp, g, slice_, eps, None, 0.5, None, 0.1, None, None, None,
                                           1, 0, 0, None)
    codes["nuts_step"] = lib.bjx_nuts_step(h, keys, q, logp, g, q, logp, g, eps, None, 2, None, None, None)
    gist = _lib.GistParams(_lib.GIST_TRAJECTORY_LENGTH, 0.5, 8, 0, 0, _lib.GIST_SYMMETRIC)
    # every native loop, then the argument checks each runs before or after its route: num_steps = 0 and thin = 0
    sample = {
        "hmc_sample": lambda n, thin: lib.bjx_hmc_sample(h, rng_key, q, logp, g, eps, None, 2, n, 0, None, thin, None),
        "nuts_sample": lambda n, thin: lib.bjx_nuts_sample(h, rng_key, q, logp, g, eps, None, 2, n, None, thin, None,
                                                           None),
        "mclmc_sample": lambda n, thin: lib.bjx_mclmc_sample(h, rng_key, q, p, logp, g, eps, None, 1.0, None, 0.1, n,
                                                             None, thin, None),
        "adjusted_mclmc_sample": lambda n, thin: lib.bjx_adjusted_mclmc_sample(
            h, rng_key, q, logp, g, eps, None, 1.0, _lib.AMCLMC_STEPS_FIXED, 2, 1.0, 1, None, n, None, thin, None, None),
        "gist_sample": lambda n, thin: lib.bjx_gist_sample(h, C.byref(gist), rng_key, q, logp, g, eps, None, n, None,
                                                           thin, None, None),
        "mala_sample": lambda n, thin: lib.bjx_mala_sample(h, rng_key, q, logp, g, eps, None, n, None, thin, None),
        "barker_sample": lambda n, thin: lib.bjx_barker_sample(h, rng_key, q, logp, g, eps, None, n, None, thin, None),
        "elliptical_slice_sample": lambda n, thin: lib.bjx_elliptical_slice_sample(h, rng_key, q, logp, n, 8, None,
                                                                                   thin, None),
    }
    for name in ("hmc_sample", "nuts_sample", "mclmc_sample", "adjusted_mclmc_sample", "gist_sample", "mala_sample",
                 "barker_sample"):
        codes[name] = sample[name](4, 1)
    # no prior yet on the handle's first integrator; the second finds the one set below
    codes["elliptical_slice_sample_no_prior"] = sample["elliptical_slice_sample"](4, 1)
    # a dense metric grid point takes the dense prior: the small matvec, the tensor-core product or its refusal
    dense = metric == "dense"
    codes["set_elliptical_prior"] = lib.bjx_set_elliptical_prior(
        h, _lib.METRIC_DENSE if dense else _lib.METRIC_DIAG, dev(np.zeros(D)), dev(np.eye(D) if dense else np.ones(D)))
    codes["elliptical_slice_sample"] = sample["elliptical_slice_sample"](4, 1)
    for name, call in sample.items():
        codes[f"{name}_num_steps_0"] = call(0, 1)
        codes[f"{name}_thin_0"] = call(4, 0)
    codes["synchronize"] = lib.bjx_synchronize(h)
    return codes


def routing_codes():
    """{"target/dim/metric/integrator": {entry point: return code}} over the whole grid."""
    lib = _lib.lib()
    out = {}
    for target in TARGETS:
        for D in DIMS:
            for metric in METRICS:
                dev, rs = _Dev(), np.random.default_rng(D)
                cfg = _lib.Config()
                cfg.device, cfg.n_chains, cfg.dim, cfg.max_tree_depth = 0, N_CHAINS, D, 4
                cfg.target = _target(target, D, dev, rs)
                h = C.c_void_p()
                rc_create = lib.bjx_create(C.byref(cfg), C.byref(h))
                rc_metric = _set_metric(lib, h, metric, D, dev) if rc_create == 0 else None
                for integ, coef in INTEGRATORS.items():
                    codes = {"create": rc_create}
                    if rc_create == 0:
                        codes["set_metric"] = rc_metric
                        codes["set_integrator"] = lib.bjx_set_integrator(h, (C.c_float * len(coef))(*coef), len(coef))
                        codes.update(_transition_codes(lib, h, D, metric, dev, rs))
                    out[f"{target}/{D}/{metric}/{integ}"] = codes
                if rc_create == 0:
                    assert lib.bjx_destroy(h) == 0
    return out


def test_every_entry_point_keeps_its_route():
    with open(GOLDEN) as f:
        want = json.load(f)
    got = routing_codes()
    assert sorted(got) == sorted(want)
    diff = {k: (want[k], v) for k, v in got.items() if v != want[k]}
    assert not diff, f"return codes that changed, (golden, now): {diff}"
