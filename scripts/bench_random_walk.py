"""Random-walk Metropolis: ms per transition of all chains in the native loop (bjx_rw_sample, keep_history=False),
chain-dims per second, the acceptance rate, and the HBM bytes per transition of the model below over the time (the
share of the 3.35 TB/s data-sheet bandwidth those bytes would take).  Workloads:
  - diag_128: 65536 x 128 (config 3's shape) on a diagonal Gaussian of scales 0.5 ... 2, the additive step
    normal(2.4 / sqrt(D) * scales), on the warp rows;
  - hier_logit_10000: config 5's hierarchical logistic regression at 32768 x 10000 on the CTA rows, the additive step
    normal(0.002).
Beside each, the same number of standard normals drawn by the library's own device PRNG (bj.random.normal, per-chain
keys, written to a [C, D] array): the threefry-and-erfinv floor of the proposal, measured in the same call.
HBM model per transition (the native loop keeps no history):
  - warp rows: the state stays in registers, so the transition moves only its acceptance rate (4 B per chain) and the
    step key; the state's load and store (2 C D 4 B) are spread over the call's steps;
  - CTA rows: x is read from its row (4 D B per chain) and written back on acceptance (4 D B per accepted chain), plus
    the acceptance rate; the target's data (0.65 MB) stays in L2.
The card's name and power limit are read in the same call.  CUDA events around `steps` transitions after a warm-up of
the same shape; two rounds, the faster reported.
usage: python scripts/bench_random_walk.py [steps]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import blackjax_b200 as bj  # noqa: E402
from blackjax_b200.mcmc import random_walk as rw  # noqa: E402

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 50
dev = "cuda:0"
HBM_BYTES_PER_S = 3.35e12


def smi(query):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        return "unknown"


def timed(fn, n):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def hbm_bytes(C, D, big, acc_rate):
    """The model above: HBM bytes of one transition of all C chains."""
    if big:
        return C * D * 4 * (1.0 + acc_rate) + C * 4 + 8
    return C * 4 + 8 + 2 * C * D * 4 / steps


def workload(name, tgt, q0, prop):
    C, D = q0.shape
    st = rw.init(q0, tgt)
    key = torch.tensor([0, 7], dtype=torch.int32, device=dev).view(torch.uint32)
    acc = []

    def native():
        acc.append(bj.sample_random_walk_native(key, st, tgt, steps, proposal=prop, keep_history=False)[2])

    ms = min(timed(native, steps) for _ in range(2))
    a = float(acc[-1].double().mean())
    keys = bj.random.split(bj.random.key(3, device=dev), C)

    def normals():
        for _ in range(steps):
            bj.random.normal(keys, (D,))  # discarded: the allocator reuses the block

    ms_normals = min(timed(normals, steps) for _ in range(2))
    b = hbm_bytes(C, D, D > 1024, a)
    return {"name": name, "C": C, "D": D, "ms_per_transition": ms, "chain_dims_per_s": C * D / (ms * 1e-3),
            "acceptance_rate": a, "ms_per_C_x_D_normals": ms_normals, "hbm_bytes_per_transition_model": b,
            "hbm_share_of_3p35_TBps": b / (ms * 1e-3) / HBM_BYTES_PER_S}


def main():
    out = {"gpu": smi("name"), "power_limit_w": smi("power.limit"), "max_sm_clock_mhz": smi("clocks.max.sm"),
           "steps": steps, "workloads": []}
    C, D = 65536, 128
    s = np.geomspace(0.5, 2.0, D).astype(np.float32)
    sd = torch.tensor(s, device=dev)
    q0 = torch.randn(C, D, device=dev) * sd
    out["workloads"].append(workload("diag_128", bj.targets.DiagGaussian(s), q0,
                                     rw.normal(sd * float(2.4 / np.sqrt(D)))))
    del q0
    torch.cuda.empty_cache()
    C, D = 32768, 10000
    x, bits = bj.targets.HierLogit.synthetic_data(D - 4, seed=1)
    q0 = torch.empty(C, D, device=dev)
    q0[:, 0], q0[:, 1], q0[:, 2], q0[:, 3] = 0.5, float(np.log(0.7)), 1.0, -0.5
    q0[:, 4:] = 0.5 + 0.7 * torch.randn(C, D - 4, device=dev)
    out["workloads"].append(workload("hier_logit_10000", bj.targets.HierLogit(x, bits), q0, rw.normal(0.002)))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
