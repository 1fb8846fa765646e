"""Adjusted MCLMC's tuner (bjx_adjusted_mclmc_find_l_and_step_size) on a diagonal Gaussian with scales over two decades,
isokinetic mclachlan, for the dynamic uniform rule and the static kernel.  Reports, with the card's name and power limit:
* the time of each stage, from CUDA events around tuner runs that stop after pass 1 (frac_tune2 = 0), after both passes and
  after stage 3, each timed after a warm-up run of the same shape;
* the time per tuning step (bjx_adjusted_mclmc_tune_step, dual averaging on, mask = 1; and mask = 0, which adds the moment
  rows) against bjx_adjusted_mclmc_step transitions replayed with the same per-chain step counts;
* stage 3's per-chain ESS per transition (mean over dimensions) of the tuned chains.
usage: python scripts/bench_adjusted_mclmc_tuning.py [C] [D] [num_steps] [slice_chains]"""
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import blackjax_b200 as bj
from blackjax_b200 import _engine, _lib
from blackjax_b200.adaptation import adjusted_mclmc_adaptation as ama
from blackjax_b200.mcmc import adjusted_mclmc_dynamic as amd
from blackjax_b200.mcmc import integrators

C = int(sys.argv[1]) if len(sys.argv) > 1 else 65536
D = int(sys.argv[2]) if len(sys.argv) > 2 else 1024
N = int(sys.argv[3]) if len(sys.argv) > 3 else 1000
SLICE = int(sys.argv[4]) if len(sys.argv) > 4 else 4096
STEPS = 20  # tuning steps timed one by one
dev = "cuda:0"


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = "unknown"
    return name, out


def events():
    return torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)


tgt = bj.targets.DiagGaussian(np.logspace(-1, 1, D))
key = bj.random.key(3, dev)
q0 = bj.random.normal(bj.random.split(bj.random.key(7, dev), C), (D,))
history_bytes = SLICE * D * 4 * int(N * 0.1)


def setup(dynamic):
    if dynamic:
        st = amd.init(q0, tgt, bj.random.key(9, dev))
        return st, bj.adjusted_mclmc_dynamic.build_kernel(
            integration_steps_fn=amd.make_random_trajectory_length_fn(True, min_steps=0)), 0.65
    return bj.adjusted_mclmc.init(q0, tgt), bj.adjusted_mclmc.build_kernel(), 0.9


def timed(st, kernel, target, f2, f3, reps=2):
    def run():
        return bj.adjusted_mclmc_find_L_and_step_size(kernel, tgt, N, st, key, target, frac_tune2=f2, frac_tune3=f3,
                                                      max_history_bytes=history_bytes)
    run()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        e0, e1 = events()
        e0.record()
        res = run()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) * 1e-3)
    return float(np.median(out)), res


def step_vs_transition(st, kernel, target, mask):
    """STEPS tuning steps from the entry parameters, then the same number of plain transitions replayed with each step's
    per-chain step counts (mean ms per step of each)."""
    eng = _engine.get_engine(st.position, tgt, divergence_threshold=kernel.divergence_threshold)
    eng.set_integrator(integrators.as_coefficients(integrators.isokinetic_mclachlan))
    eng.ensure_metric(torch.ones(D, device=dev), diagonal_only=True)
    state = [t.clone() for t in st]
    eps = torch.full((C,), 0.2 * math.sqrt(D), device=dev)
    L = 2.0 * eps
    da = torch.empty(C, 5, device=dev)
    _lib.check(_lib.lib().bjx_da_init(eng.h, _lib.ptr(da), _lib.ptr(eps), None), eng.h)
    total = torch.zeros(C, device=dev)
    moments = torch.zeros(C, 2, D, device=dev)
    keys = bj.random.split(key, STEPS)
    steps, t_tune = [], 0.0
    for t in range(STEPS + 1):
        e0, e1 = events()
        e0.record()
        _, n = ama.tune_step_(eng, keys[t % STEPS], state, eps, L, da, (total, moments), None, mask, True, target,
                              device_rule=kernel.device_rule)
        e1.record()
        torch.cuda.synchronize()
        if t > 0:  # the first is a warm-up
            t_tune += e0.elapsed_time(e1)
            steps.append(n.clone())
    q, logp, g = (x.clone() for x in st[:3])
    eps_fixed = eps.clone()
    t_tr = 0.0
    for t in range(STEPS + 1):
        n = steps[max(t - 1, 0)]
        e0, e1 = events()
        e0.record()
        eng.adjusted_mclmc_step(keys[t % STEPS], q, logp, g, eps_fixed, n, math.inf, out=(q, logp, g))
        e1.record()
        torch.cuda.synchronize()
        if t > 0:
            t_tr += e0.elapsed_time(e1)
    mean_steps = float(torch.stack(steps).float().mean())
    return t_tune / STEPS, t_tr / STEPS, mean_steps


res = {"C": C, "D": D, "num_steps": N, "stage3_slice_chains": SLICE}
n1, n2, n3 = ama.stage_lengths(N, 0.1, 0.1, 0.1)
res["stages"] = {"n1": n1, "n2": n2, "n3": n3}
for label, dynamic in (("dynamic_uniform", True), ("static", False)):
    st, kernel, target = setup(dynamic)
    t1, _ = timed(st, kernel, target, 0.0, 0.0)
    t12, _ = timed(st, kernel, target, 0.1, 0.0)
    t123, (fin, par, count) = timed(st, kernel, target, 0.1, 0.1)
    assert bool(torch.isfinite(par.step_size).all()) and bool(torch.isfinite(par.L).all())
    tm1, tr1, ms1 = step_vs_transition(st, kernel, target, 1)
    tm0, tr0, ms0 = step_vs_transition(st, kernel, target, 0)
    # stage 3's ESS per transition at the tuned parameters, on one slice
    n = min(SLICE, C)
    avg = (par.L / par.step_size)[:n].contiguous()
    sub = type(fin)(*(t[:n].clone() for t in fin))
    kw = (dict(integration_steps_fn=amd.make_random_trajectory_length_fn(True, min_steps=0),
               integration_steps_params=(avg,)) if dynamic else dict(num_integration_steps=avg))
    _, hist, _, _ = bj.sample_adjusted_mclmc_native(key, sub, tgt, par.step_size[:n].contiguous(), n3,
                                                    inverse_mass_matrix=par.inverse_mass_matrix[:n].contiguous(), **kw)
    ess = bj.diagnostics.effective_sample_size(hist, tgt, per_chain=True)
    r = (ess.mean(1) / n3).cpu().numpy()
    res[label] = {"pass1_s": round(t1, 4), "pass2_s": round(t12 - t1, 4), "stage3_s": round(t123 - t12, 4),
                  "total_s": round(t123, 4),
                  "ms_per_tuning_step_mask1": round(tm1, 3), "ms_per_transition_same_steps_mask1": round(tr1, 3),
                  "mean_steps_mask1": round(ms1, 3),
                  "ms_per_tuning_step_mask0": round(tm0, 3), "ms_per_transition_same_steps_mask0": round(tr0, 3),
                  "mean_steps_mask0": round(ms0, 3),
                  "stage3_ess_per_transition": {"median": float(np.median(r)), "min": float(r.min()),
                                                "max": float(r.max())},
                  "L_over_step_median": float(torch.median(par.L / par.step_size))}
name, pl = card()
res["card"], res["power_limit_and_max_sm_clock"] = name, pl
print(json.dumps(res))
