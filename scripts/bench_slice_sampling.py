"""Slice sampling: ms per transition of all chains, the mean number of target evaluations per transition (counted on the
device) and the target evaluations per second.  Workloads:
  - diag_1024: 65536 x 1024, a diagonal Gaussian (scales 0.1 ... 10) with the direction scale [D] = the scales, under
    both intervals: the native loop (bjx_slice_sample, one persistent launch) against the step API (one launch per
    transition), alternating rounds;
  - hier_logit_10000: BASELINE config 5's hierarchical logistic regression at 32768 x 10000 on the CTA rows (doubling);
  - ess_diag_1024: elliptical slice sampling on the same 65536 x 1024 shape (a diagonal Gaussian likelihood of scales
    0.1 ... 10 under the prior N(0, I)), the sibling sampler, in the same run.
Every chain starts at an exact draw of its target.  The targets also form the gradient, which both samplers discard.
The card's name, power limit and max SM clock are read in the same call.  CUDA events around `steps` transitions after
a warm-up of the same shape; two rounds, the faster reported.
usage: python scripts/bench_slice_sampling.py [steps]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import blackjax_b200 as bj  # noqa: E402
from blackjax_b200.mcmc import slice as sl  # noqa: E402

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
dev = "cuda:0"


def smi(query):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        return "unknown"


def timed(fn):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def slice_workload(name, C, D, tgt, scale, q0, interval, step_api):
    st = sl.init(q0, tgt)
    key = torch.tensor([0, 7], dtype=torch.int32, device=dev).view(torch.uint32)
    ev = torch.zeros(1, dtype=torch.uint64, device=dev)

    def native():
        ev.zero_()
        bj.sample_slice_sampling_native(key, st, tgt, steps, scale=scale, interval=interval, keep_history=False,
                                        evaluations=ev)

    kern = sl.build_kernel(interval, inplace=True)
    prop = sl.direction_proposal(scale)
    keys = torch.randint(0, 2**31 - 1, (steps, 2), dtype=torch.int32, device=dev).view(torch.uint32)

    def steps_fn():
        s = tuple(t.clone() for t in st)
        for t in range(steps):
            kern(keys[t], s, tgt, prop)

    rounds = {"native": [], "step_api": []}
    for _ in range(2):  # alternate the two
        rounds["native"].append(timed(native))
        if step_api:
            rounds["step_api"].append(timed(steps_fn))
    ms = min(rounds["native"])
    evals = float(ev.cpu().item()) / (C * steps)
    w = {"name": name, "C": C, "D": D, "ms_per_transition": ms, "mean_evals_per_transition": evals,
         "target_evals_per_s": C * evals / (ms * 1e-3)}
    if step_api:
        w["ms_per_transition_step_api"] = min(rounds["step_api"])
    return w


def main():
    out = {"gpu": smi("name"), "power_limit_w": smi("power.limit"), "max_sm_clock_mhz": smi("clocks.max.sm"),
           "steps": steps, "workloads": []}
    C, D = 65536, 1024
    s = np.geomspace(0.1, 10.0, D).astype(np.float32)
    sd = torch.tensor(s, device=dev)
    tgt = bj.targets.DiagGaussian(s)
    for name, interval in (("diag_1024_doubling", sl.doubling), ("diag_1024_stepping_out", sl.stepping_out)):
        q0 = torch.randn(C, D, device=dev) * sd
        out["workloads"].append(slice_workload(name, C, D, tgt, sd, q0, interval, True))
        del q0
        torch.cuda.empty_cache()
    # elliptical slice sampling on the same shape
    post_sd = torch.tensor(s / np.sqrt(1.0 + s * s), device=dev)
    q0 = torch.randn(C, D, device=dev) * post_sd
    st = bj.elliptical_slice.init(q0, tgt)
    key = torch.tensor([0, 7], dtype=torch.int32, device=dev).view(torch.uint32)
    sub = []

    def ess_native():
        sub.append(bj.sample_elliptical_slice_native(key, st, tgt, 0.0, torch.ones(D, device=dev), steps,
                                                     keep_history=False)[2])

    ms = min(timed(ess_native) for _ in range(2))
    m = float(sub[-1].double().mean())
    out["workloads"].append({"name": "ess_diag_1024", "C": C, "D": D, "ms_per_transition": ms,
                             "mean_evals_per_transition": m, "target_evals_per_s": C * m / (ms * 1e-3)})
    del st, q0
    torch.cuda.empty_cache()
    C, D = 32768, 10000
    x, bits = bj.targets.HierLogit.synthetic_data(D - 4, seed=1)
    q0 = torch.empty(C, D, device=dev)
    q0[:, 0], q0[:, 1], q0[:, 2], q0[:, 3] = 0.5, float(np.log(0.7)), 1.0, -0.5
    q0[:, 4:] = 0.5 + 0.7 * torch.randn(C, D - 4, device=dev)
    out["workloads"].append(slice_workload("hier_logit_10000", C, D, bj.targets.HierLogit(x, bits), 0.5, q0,
                                           sl.doubling, False))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
