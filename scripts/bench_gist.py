"""GIST with a self-tuning trajectory length (bjx_gist_sample) against NUTS (bjx_nuts_sample) at the same step size and
metric, on two workloads: Neal's funnel at D = 128 (identity metric) and a diagonal Gaussian with scales 0.1 ... 10 at
D = 1024 (the metric a warm-up would adapt, scales^2).  C = 65536 chains by default.  Per sampler and workload: ms per
transition of all chains (CUDA events around `steps` transitions enqueued back to back, after a warm-up run of the same
shape; the two samplers alternate, two rounds each), gradient evaluations per transition and per second, and the device
ESS per second of the slowest coordinate (the funnel's neck, the Gaussian's widest scale) over the same run.  The native
loop reports L only, so GIST's mean U, L and N come from 5 step-API transitions that continue from the end of the timed
run, averaged over all chains: a transition costs about U + L + N gradient evaluations (the proposal is re-integrated
rather than cached), NUTS one per leaf of its tree (its mean tree size over the timed run).  The card's name and power
limit are read in the same call.
usage: python scripts/bench_gist.py [C] [steps]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import blackjax_b200 as bj  # noqa: E402

C = int(sys.argv[1]) if len(sys.argv) > 1 else 65536
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 20
dev = "cuda:0"
UNL_STEPS = 5


def smi(query):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        return "unknown"


def workload(name):
    if name == "funnel_128":
        D = 128
        tgt = bj.targets.Funnel(D)
        q = 0.5 * bj.random.normal(bj.random.split(bj.random.key(7, dev), C), (D,))
        return tgt, q, torch.ones(D, device=dev), 0.1, 0
    D = 1024
    scales = np.logspace(-1, 1, D).astype(np.float32)
    tgt = bj.targets.DiagGaussian(scales)
    s = torch.from_numpy(scales).to(dev)
    q = bj.random.normal(bj.random.split(bj.random.key(7, dev), C), (D,)) * s
    return tgt, q, s * s, 0.5, D - 1


def run(sampler, st, tgt, eps, imm, n):
    key = bj.random.key(3, dev)
    if sampler == "gist":
        return bj.sample_gist_native(key, st, tgt, eps, imm, n)
    return bj.sample_nuts_native(key, st, tgt, eps, imm, n)


res = {"card": torch.cuda.get_device_name(0), "power_limit_W": smi("power.limit"), "C": C, "steps": steps,
       "integrator": "velocity_verlet", "gist": {"path_fraction": 0.5, "max_num_steps": 1024},
       "nuts": {"max_num_doublings": 10}}
for wl in ("funnel_128", "diag_gaussian_1024"):
    tgt, q, imm, eps, stat = workload(wl)
    st = bj.gist_trajectory_length.init(q, tgt)
    out = {"step_size": eps, "statistic_dim": stat}
    times = {"gist": [], "nuts": []}
    last = {}
    for sampler in ("gist", "nuts"):
        run(sampler, st, tgt, eps, imm, 2)  # warm-up of the same shape
    torch.cuda.synchronize()
    for rnd in range(2):
        for sampler in ("gist", "nuts"):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = run(sampler, st, tgt, eps, imm, steps)
            e1.record()
            torch.cuda.synchronize()
            times[sampler].append(e0.elapsed_time(e1) * 1e-3 / steps)
            last[sampler] = r
    for sampler in ("gist", "nuts"):
        fin, hist, acc, n_int = last[sampler]
        t = float(np.median(times[sampler]))
        ess = float(bj.diagnostics.effective_sample_size(hist, tgt)[stat])
        d = {"ms_per_transition": round(t * 1e3, 3), "spread_ms": [round(x * 1e3, 3) for x in sorted(times[sampler])],
             "mean_acceptance": round(float(acc.mean()), 3), "ess": round(ess, 1),
             "ess_per_s": round(ess / (t * steps), 1)}
        if sampler == "gist":  # U / L / N over UNL_STEPS step-API transitions continuing from the timed run's end
            kern, cur, ul = bj.gist_trajectory_length.build_kernel(), fin, torch.zeros(3, device=dev)
            for k in range(UNL_STEPS):
                cur, info = kern(bj.random.key(100 + k, dev), cur, tgt, eps, imm)
                ul += torch.stack([x.float().mean() for x in (info.num_steps_to_uturn_forward, info.num_integration_steps,
                                                              info.num_steps_to_uturn_reverse)])
            U, L, N = (float(x) / UNL_STEPS for x in ul)
            grads = U + L + N
            d.update(mean_U=round(U, 2), mean_L=round(L, 2), mean_N=round(N, 2))
        else:
            grads = float(n_int.float().mean())
        d.update(gradient_evals_per_transition=round(grads, 2), gradient_evals_per_s=round(grads * C / t, 1))
        out[sampler] = d
    res[wl] = out
    print(f"{wl}: GIST {out['gist']['ms_per_transition']} ms/transition (U {out['gist']['mean_U']}, L "
          f"{out['gist']['mean_L']}, N {out['gist']['mean_N']}), ESS/s {out['gist']['ess_per_s']}; NUTS "
          f"{out['nuts']['ms_per_transition']} ms/transition, ESS/s {out['nuts']['ess_per_s']}")
print(f"on {res['card']} ({res['power_limit_W']} W)")
print(json.dumps(res))
