"""Adjusted MCLMC (MAMS): the native run loop (bjx_adjusted_mclmc_sample) on the diagonal Gaussian with the default
isokinetic mclachlan table: static n = 8 (L_proposal_factor 1, and inf for no momentum refresh) and the dynamic uniform rule
max(ceil(U * rescale(8)), 1).  Reports ms per transition of all chains, gradient evaluations/s (two per mclachlan step),
mean acceptance and the bytes/s equivalent of the 8 * D bytes per chain and transition the kernel has to move (q, grad
read; the accepted write-back is not counted), with the card's name, power limit and median SM clock sampled during the
run.  Each timing is over `steps` transitions enqueued back to back and ended by a device synchronise (CUDA events), after
a warm-up run of the same shape.  The same shape through bjx_mclmc_sample (one isokinetic step per transition, L = inf)
is timed beside it, for the per-step cost.
usage: python scripts/bench_adjusted_mclmc.py [C] [D] [steps]"""
import json
import os
import subprocess
import sys
import threading

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import blackjax_b200 as bj  # noqa: E402
from blackjax_b200.mcmc import adjusted_mclmc_dynamic as amd  # noqa: E402

C = int(sys.argv[1]) if len(sys.argv) > 1 else 65536
D = int(sys.argv[2]) if len(sys.argv) > 2 else 1024
steps = int(sys.argv[3]) if len(sys.argv) > 3 else 50
dev = "cuda:0"
GRADS_PER_STEP = 2  # mclachlan: two position updates, each followed by value_and_grad
AVG = 8


def smi(query):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        return "unknown"


class ClockSampler:
    """SM clock (MHz) sampled every 0.2 s while a timing runs"""

    def __init__(self):
        self.samples, self._stop = [], threading.Event()

    def __enter__(self):
        def run():
            while not self._stop.wait(0.2):
                v = smi("clocks.sm")
                if v.isdigit():
                    self.samples.append(int(v))
        self._t = threading.Thread(target=run, daemon=True)
        self._t.start()
        return self

    def __exit__(self, *a):
        self._stop.set()
        self._t.join()


scales = np.logspace(-1, 1, D)
tgt = bj.targets.DiagGaussian(scales)
key = bj.random.key(3, dev)
q0 = bj.random.normal(bj.random.split(bj.random.key(7, dev), C), (D,)) * torch.from_numpy(scales.astype(np.float32)).to(dev)
imm = torch.from_numpy(scales.astype(np.float32) ** 2).to(dev)
eps = float(np.sqrt(D)) * 0.5
st = bj.adjusted_mclmc.init(q0, tgt)
dst = bj.adjusted_mclmc_dynamic.init(q0, tgt, bj.random.key(11, dev))
uniform_rule = amd.make_random_trajectory_length_fn(True)


def run(kind, n):
    if kind.startswith("static"):
        return bj.sample_adjusted_mclmc_native(key, st, tgt, eps, n, num_integration_steps=AVG,
                                               L_proposal_factor=float("inf") if kind.endswith("no_refresh") else 1.0,
                                               inverse_mass_matrix=imm, keep_history=False)
    if kind == "dynamic":
        return bj.sample_adjusted_mclmc_native(key, dst, tgt, eps, n, integration_steps_fn=uniform_rule,
                                               integration_steps_params=(AVG,), L_proposal_factor=1.0,
                                               inverse_mass_matrix=imm, keep_history=False)
    mst = bj.mclmc.init(q0, tgt, key)
    return bj.sample_mclmc_native(key, mst, tgt, float("inf"), eps, n, inverse_mass_matrix=imm, keep_history=False)


def timed(kind):
    """median seconds per transition over three runs of `steps` transitions, after a warm-up run of the same shape"""
    run(kind, 5)
    torch.cuda.synchronize()
    out, clocks, extra = [], [], {}
    for rep in range(3):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with ClockSampler() as cs:
            e0.record()
            res = run(kind, steps)
            e1.record()
            torch.cuda.synchronize()
        clocks += cs.samples
        out.append(e0.elapsed_time(e1) * 1e-3 / steps)
    if kind != "mclmc":
        _, _, acc, n_hist = res
        extra = {"mean_acceptance": round(float(acc.mean()), 3), "mean_steps": round(float(n_hist.float().mean()), 3)}
        assert bool(torch.isfinite(res[0].position).all())
    else:
        extra = {"mean_steps": 1.0}
    return float(np.median(out)), [round(x * 1e3, 3) for x in sorted(out)], clocks, extra


name, pl = torch.cuda.get_device_name(0), smi("power.limit")
res = {"card": name, "power_limit_W": pl, "C": C, "D": D, "steps": steps, "target": "diag_gaussian",
       "integrator": "isokinetic_mclachlan"}
all_clocks = []
for kind in ("static", "static_no_refresh", "dynamic", "mclmc"):
    t, spread, clocks, extra = timed(kind)
    all_clocks += clocks
    grads = GRADS_PER_STEP * extra["mean_steps"] * C / t
    res[kind] = {"ms_per_transition": round(t * 1e3, 3), "spread_ms": spread, "gradient_evals_per_s": round(grads, 1),
                 "ms_per_integration_step": round(t * 1e3 / extra["mean_steps"], 3),
                 "equivalent_GB_per_s_at_8D": round(8.0 * D * C / t / 1e9, 1), **extra}
res["median_sm_clock_MHz"] = int(np.median(all_clocks)) if all_clocks else "unknown"
print(f"adjusted MCLMC C={C} D={D} on {name} ({pl} W, median SM clock {res['median_sm_clock_MHz']} MHz): "
      f"static n={AVG}: {res['static']['ms_per_transition']} ms/transition, acceptance {res['static']['mean_acceptance']}; "
      f"dynamic avg {AVG}: {res['dynamic']['ms_per_transition']} ms/transition; "
      f"static without refresh: {res['static_no_refresh']['ms_per_integration_step']} ms/step; "
      f"MCLMC (1 step, L = inf): {res['mclmc']['ms_per_transition']} ms/transition")
print(json.dumps(res))
