"""MCLMC: the native run loop (bjx_mclmc_sample) on the diagonal Gaussian with the default isokinetic mclachlan table.
Reports transitions/s, gradient evaluations/s (two per mclachlan transition) and the HBM share of the transition from
24 * D bytes per chain (q, p, grad read and written; the log-density and the per-chain scalars are not counted) against the
H100 SXM data sheet's 3.35 TB/s, with the card's name and power limit.  Each timing is over `steps` transitions enqueued
back to back and ended by a device synchronise (CUDA events), after a warm-up run of the same shape.  The same run with
L = inf, which skips the two partial momentum refreshes, is timed first for comparison.
usage: python scripts/bench_mclmc.py [C] [D] [steps]"""
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import blackjax_b200 as bj

C = int(sys.argv[1]) if len(sys.argv) > 1 else 65536
D = int(sys.argv[2]) if len(sys.argv) > 2 else 1024
steps = int(sys.argv[3]) if len(sys.argv) > 3 else 200
dev = "cuda:0"
PEAK_HBM = 3.35e12
GRADS_PER_TRANSITION = 2  # mclachlan: two position updates, each followed by value_and_grad


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        pl = "unknown"
    return name, pl


tgt = bj.targets.DiagGaussian(np.logspace(-1, 1, D))
key = bj.random.key(3, dev)
q0 = bj.random.normal(bj.random.split(bj.random.key(7, dev), C), (D,))
imm = torch.from_numpy(np.logspace(-1, 1, D).astype(np.float32) ** 2).to(dev)
st = bj.mclmc.init(q0, tgt, key)
L, eps = math.sqrt(D), 0.3 * math.sqrt(D)


def timed(L_run):
    """median seconds per transition over three runs of `steps` transitions, after a warm-up run of the same shape"""
    bj.sample_mclmc_native(key, st, tgt, L_run, eps, 10, inverse_mass_matrix=imm, keep_history=False)
    torch.cuda.synchronize()
    out = []
    for rep in range(3):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fin, _, de = bj.sample_mclmc_native(key, st, tgt, L_run, eps, steps, inverse_mass_matrix=imm, keep_history=False)
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) * 1e-3 / steps)
    assert bool(torch.isfinite(fin.position).all()) and bool(torch.isfinite(de).all())
    return out


# L = inf skips both partial refreshes (integrators.py:569-572): the difference is the cost of the 2 D normal draws and
# the two renormalisations per chain and transition
times_no_refresh = timed(math.inf)
times = timed(L)
t = float(np.median(times))
name, pl = card()
res = {"card": name, "power_limit": pl, "C": C, "D": D, "steps": steps, "target": "diag_gaussian",
       "integrator": "isokinetic_mclachlan", "us_per_transition": round(t * 1e6, 1),
       "transitions_per_s": round(C / t, 1), "gradient_evals_per_s": round(GRADS_PER_TRANSITION * C / t, 1),
       "hbm_share": round(24.0 * D * C / t / PEAK_HBM, 3), "spread_us": [round(x * 1e6, 1) for x in sorted(times)],
       "us_per_transition_without_refresh": round(float(np.median(times_no_refresh)) * 1e6, 1)}
print(f"MCLMC C={C} D={D} on {name} ({pl}): {res['us_per_transition']} us per transition of all chains, "
      f"{res['transitions_per_s']:.3g} chain transitions/s, {res['gradient_evals_per_s']:.3g} gradients/s, "
      f"{100 * res['hbm_share']:.1f} % of 3.35 TB/s; with L = inf (no momentum refresh) "
      f"{res['us_per_transition_without_refresh']} us")
print(json.dumps(res))
