"""MALA and Barker's proposal: ms per transition of all chains through the step API (one launch per transition, enqueued
back to back) and through the native loop (bjx_mala_sample / bjx_barker_sample: one launch for all transitions), with
HMC at L = 1 on the same shape as the one-gradient anchor.  Workloads: MALA on Neal's funnel at 65536 x 128, Barker with
a diagonal metric on a diagonal Gaussian with scales 0.1 ... 10 at 65536 x 1024, and MALA on the hierarchical logistic
regression of BASELINE config 5 at 32768 x 10000 (the CTA-per-chain rows), each from a start in the target's bulk at a
step size with a moderate acceptance rate.  The step kernel's bytes/s counts the (q, grad) rows read, the proposal's
(position, grad) rows Barker's step API writes as info, and, at the measured acceptance rate, the (q, grad) rows written,
over its time, against the H100 SXM's 3.35 TB/s.  The
card's name, power limit and max SM clock are read in the same call.  CUDA events around `steps` transitions after a
warm-up of the same shape; the variants alternate over two rounds and the faster round is reported.
usage: python scripts/bench_langevin.py [steps]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import blackjax_b200 as bj  # noqa: E402

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 50
dev = "cuda:0"
HBM = 3.35e12


def smi(query):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        return "unknown"


def workload(name):
    if name == "mala_funnel_128":
        C, D = 65536, 128
        q0 = torch.randn(C, D, device=dev)
        q0[:, 0] = 0.0  # the funnel's bulk at the neck y = 0
        return "mala", C, D, bj.targets.Funnel(D), 0.1, None, q0
    if name == "barker_diag_1024":
        C, D = 65536, 1024
        s = np.geomspace(0.1, 10.0, D).astype(np.float32)
        # M^1/2 = sqrt(1 / M^-1) = s: the proposal moves each coordinate on its own scale
        q0 = torch.randn(C, D, device=dev) * torch.tensor(s, device=dev)
        return "barker", C, D, bj.targets.DiagGaussian(s), 0.5, torch.tensor(1.0 / (s * s), device=dev), q0
    C, D = 32768, 10000
    x, bits = bj.targets.HierLogit.synthetic_data(D - 4, seed=1)
    # a start in the typical set: the data-generating values and N(0.5, 0.7^2) group effects
    q0 = torch.empty(C, D, device=dev)
    q0[:, 0], q0[:, 1], q0[:, 2], q0[:, 3] = 0.5, float(np.log(0.7)), 1.0, -0.5
    q0[:, 4:] = 0.5 + 0.7 * torch.randn(C, D - 4, device=dev)
    return "mala", C, D, bj.targets.HierLogit(x, bits), 1e-4, None, q0


def timed(fn):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    out = {"gpu": smi("name"), "power_limit_w": smi("power.limit"), "max_sm_clock_mhz": smi("clocks.max.sm"),
           "steps": steps, "workloads": []}
    for name in ("mala_funnel_128", "barker_diag_1024", "mala_hier_logit_10000"):
        sampler, C, D, tgt, eps, imm, q0 = workload(name)
        st = bj.mala.init(q0, tgt)
        key = torch.tensor([0, 7], dtype=torch.int32, device=dev).view(torch.uint32)
        keys = torch.randint(0, 2**31 - 1, (steps, 2), dtype=torch.int32, device=dev).view(torch.uint32)
        mod = bj.mala if sampler == "mala" else bj.barker
        kern = mod.build_kernel(inplace=True)
        hmc = bj.hmc.build_kernel(inplace=True)
        imm_h = imm if imm is not None else torch.ones(D, device=dev)
        acc = []

        def step_api():
            s = tuple(t.clone() for t in st)
            for t in range(steps):
                args = (eps,) if sampler == "mala" else (eps, imm)
                _, info = kern(keys[t], s, tgt, *args)
            acc.append(info.acceptance_rate)  # read after the timed window

        def native():
            fn = bj.sample_mala_native if sampler == "mala" else bj.sample_barker_native
            extra = () if sampler == "mala" else (imm,)
            fn(key, st, tgt, eps, steps, *extra, keep_history=False)

        def hmc_l1():
            s = tuple(t.clone() for t in st)
            for t in range(steps):
                hmc(keys[t], s, tgt, eps, imm_h, 1)

        res = {k: [] for k in ("step", "native", "hmc_L1")}
        for _ in range(2):
            res["step"].append(timed(step_api))
            res["native"].append(timed(native))
            res["hmc_L1"].append(timed(hmc_l1))
        ms = {k: min(v) for k, v in res.items()}
        a = float(acc[-1].mean())
        # read (q, grad), write them on acceptance; Barker's step API also writes the proposal's (position, grad)
        nbytes = 4.0 * C * D * (2 + 2 * a + (2 if sampler == "barker" else 0))
        out["workloads"].append({"name": name, "C": C, "D": D, "sampler": sampler, "ms_per_transition_step": ms["step"],
                                 "ms_per_transition_native": ms["native"], "ms_per_transition_hmc_L1": ms["hmc_L1"],
                                 "acceptance": a, "step_bytes_per_s": nbytes / (ms["step"] * 1e-3),
                                 "step_share_of_hbm": nbytes / (ms["step"] * 1e-3) / HBM})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
