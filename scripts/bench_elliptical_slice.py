"""Elliptical slice sampling: ms per transition of all chains through the native loop (bjx_elliptical_slice_sample), the
mean number of likelihood evaluations per transition (subiter) and the likelihood evaluations per second.  Workloads:
  - diag_1024: 65536 x 1024, a diagonal Gaussian likelihood (scales 0.5 ... 2) under the prior N(0, I): the warp rows,
    one persistent launch for all transitions, and for comparison the step API (one launch per transition);
  - se_kernel_1024: 65536 x 1024, a Gaussian-process prior with the squared-exponential kernel (length scale 0.1) on
    1024 grid points of [0, 1] plus 1e-3 jitter, and a diagonal Gaussian likelihood of noise 0.3 around a smooth curve:
    the tensor-core route, three launches per transition (normal draw, product, slice kernel).  A profiled run of its own
    gives the share of the draw and of the product (the operand split and the GEMM) in the transition's kernel time;
  - hier_logit_10000: BASELINE config 5's hierarchical logistic regression as the likelihood at 32768 x 10000 under the
    prior N(0, I) on the CTA rows.
Every chain starts in the bulk of its posterior.  The targets also form the gradient, which elliptical slice sampling
discards: a known cost of these numbers.  The card's name, power limit and max SM clock are read in the same call.
CUDA events around `steps` transitions after a warm-up of the same shape; two rounds, the faster reported.
usage: python scripts/bench_elliptical_slice.py [steps]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import blackjax_b200 as bj  # noqa: E402

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
dev = "cuda:0"


def smi(query):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        return "unknown"


def workload(name):
    if name == "diag_1024":
        C, D = 65536, 1024
        s = np.geomspace(0.5, 2.0, D).astype(np.float32)
        post_sd = torch.tensor(s / np.sqrt(1.0 + s * s), device=dev)  # N(0, 1) prior times N(0, s^2) likelihood
        return C, D, bj.targets.DiagGaussian(s), 0.0, torch.ones(D, device=dev), torch.randn(C, D, device=dev) * post_sd
    if name == "se_kernel_1024":
        C, D = 65536, 1024
        x = np.linspace(0.0, 1.0, D)
        K = np.exp(-0.5 * ((x[:, None] - x[None, :]) / 0.1) ** 2) + 1e-3 * np.eye(D)
        y = np.sin(6.0 * x).astype(np.float32)
        tgt = bj.targets.DiagGaussian(np.full(D, 0.3), mean=y)
        return C, D, tgt, 0.0, torch.tensor(K, dtype=torch.float32, device=dev), torch.tensor(y, device=dev).repeat(C, 1)
    C, D = 32768, 10000
    x, bits = bj.targets.HierLogit.synthetic_data(D - 4, seed=1)
    q0 = torch.empty(C, D, device=dev)
    q0[:, 0], q0[:, 1], q0[:, 2], q0[:, 3] = 0.5, float(np.log(0.7)), 1.0, -0.5
    q0[:, 4:] = 0.5 + 0.7 * torch.randn(C, D - 4, device=dev)
    return C, D, bj.targets.HierLogit(x, bits), 0.0, torch.ones(D, device=dev), q0


def timed(fn):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def kernel_shares(fn):
    """Share of the tensor-core route's kernel time per stage, from a torch.profiler run of fn."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    t = {}
    for e in prof.key_averages():
        if e.device_type.name != "CUDA":
            continue
        n = e.key
        stage = ("draw" if "k_dense_normal" in n else "slice" if "k_ess_transition" in n
                 else "split" if "split2" in n else "product" if "gemm" in n.lower() else "other")
        t[stage] = t.get(stage, 0.0) + e.device_time_total
    tot = sum(t.values())
    return {k: v / tot for k, v in t.items()} if tot > 0 else {}


def main():
    out = {"gpu": smi("name"), "power_limit_w": smi("power.limit"), "max_sm_clock_mhz": smi("clocks.max.sm"),
           "steps": steps, "workloads": []}
    for name in ("diag_1024", "se_kernel_1024", "hier_logit_10000"):
        C, D, tgt, mean, cov, q0 = workload(name)
        st = bj.elliptical_slice.init(q0, tgt)
        key = torch.tensor([0, 7], dtype=torch.int32, device=dev).view(torch.uint32)
        sub = []

        def native():
            _, _, s = bj.sample_elliptical_slice_native(key, st, tgt, mean, cov, steps, keep_history=False)
            sub.append(s)

        ms = min(timed(native) for _ in range(2))
        mean_sub = float(sub[-1].double().mean())
        w = {"name": name, "C": C, "D": D, "ms_per_transition": ms, "mean_subiter": mean_sub,
             "likelihood_evals_per_s": C * mean_sub / (ms * 1e-3)}
        if name == "diag_1024":
            kern = bj.elliptical_slice.build_kernel(cov, mean, inplace=True)
            keys = torch.randint(0, 2**31 - 1, (steps, 2), dtype=torch.int32, device=dev).view(torch.uint32)

            def step_api():
                s = tuple(t.clone() for t in st)
                for t in range(steps):
                    kern(keys[t], s, tgt)

            w["ms_per_transition_step_api"] = min(timed(step_api) for _ in range(2))
        if name == "se_kernel_1024":
            try:
                w["kernel_time_shares"] = kernel_shares(native)
            except Exception as e:  # the timings above stand without the profile
                w["kernel_time_shares"] = f"not measured: {e!r}"
        out["workloads"].append(w)
        del st, q0
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
