"""MCLMC's tuner (bjx_mclmc_find_l_and_step_size) on the diagonal Gaussian with the isokinetic mclachlan table.
Reports, with the card's name and power limit:
* the time of each stage, from CUDA events around three tuner runs that stop after stage 1, after stages 1-2 (with the
  readjustment) and after stage 3, each timed after a warm-up run of the same shape;
* the time per tuning step (stage 1 over its n1 steps) against bjx_mclmc_sample's time per transition at the tuned-from
  parameters;
* the per-chain ESS kernel alone on a [n3, slice, D] position history of plain MCLMC draws, and the lags it evaluated.
usage: python scripts/bench_mclmc_tuning.py [C] [D] [num_steps] [slice_chains]"""
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import blackjax_b200 as bj
from blackjax_b200 import _lib
from blackjax_b200.adaptation import mclmc_adaptation as ma

C = int(sys.argv[1]) if len(sys.argv) > 1 else 65536
D = int(sys.argv[2]) if len(sys.argv) > 2 else 1024
N = int(sys.argv[3]) if len(sys.argv) > 3 else 2000
SLICE = int(sys.argv[4]) if len(sys.argv) > 4 else 4096
dev = "cuda:0"


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = "unknown"
    return name, out


tgt = bj.targets.DiagGaussian(np.logspace(-1, 1, D))
key = bj.random.key(3, dev)
q0 = bj.random.normal(bj.random.split(bj.random.key(7, dev), C), (D,))
st = bj.mclmc.init(q0, tgt, key)
kernel = bj.mclmc.build_kernel()
history_bytes = SLICE * D * 4 * round(N * 0.1)


def timed(f1, f2, f3, reps=2):
    def run():
        return ma.mclmc_find_L_and_step_size(kernel, N, st, key, tgt, frac_tune1=f1, frac_tune2=f2, frac_tune3=f3,
                                             max_history_bytes=history_bytes)
    run()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _, par, _ = run()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) * 1e-3)
    return float(np.median(out)), par


n1, n2, r, n3, count = ma.stage_lengths(N, 0.1, 0.1, 0.1, True)
t1, _ = timed(0.1, 0.0, 0.0)
t12, _ = timed(0.1, 0.1, 0.0)
t123, par = timed(0.1, 0.1, 0.1)
assert bool(torch.isfinite(par.step_size).all()) and bool(torch.isfinite(par.L).all())

# plain transitions at the initial parameters, per step
L0, eps0 = math.sqrt(D), 0.25 * math.sqrt(D)
bj.sample_mclmc_native(key, st, tgt, L0, eps0, 10, keep_history=False)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
bj.sample_mclmc_native(key, st, tgt, L0, eps0, n1, keep_history=False)
e1.record()
torch.cuda.synchronize()
t_sample = e0.elapsed_time(e1) * 1e-3 / n1

# the per-chain ESS alone on one stage-3 slice of draws
sub = bj.mcmc.hmc.IntegratorState(*(t[:SLICE].clone() for t in st))
sub_tgt = tgt
_, hist, _ = bj.sample_mclmc_native(key, sub, sub_tgt, par.L[:SLICE].contiguous(), par.step_size[:SLICE].contiguous(),
                                    n3, inverse_mass_matrix=par.inverse_mass_matrix[:SLICE].contiguous())
eng = bj._engine.get_engine(hist[0], sub_tgt)
ess = torch.empty(SLICE, D, dtype=torch.float32, device=dev)
lags = torch.zeros(SLICE, dtype=torch.int32, device=dev)
for _ in range(2):
    _lib.check(_lib.lib().bjx_mclmc_ess_per_chain(eng.h, _lib.ptr(hist), n3, _lib.ptr(ess), _lib.ptr(lags)), eng.h)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(5):
    _lib.check(_lib.lib().bjx_mclmc_ess_per_chain(eng.h, _lib.ptr(hist), n3, _lib.ptr(ess), _lib.ptr(lags)), eng.h)
e1.record()
torch.cuda.synchronize()
t_ess = e0.elapsed_time(e1) * 1e-3 / 5
lag_np = lags.cpu().numpy()

name, pl = card()
res = {"card": name, "power_limit_and_max_sm_clock": pl, "C": C, "D": D, "num_steps": N,
       "stages": {"n1": n1, "n2": n2, "readjust": r, "n3": n3}, "stage3_slice_chains": SLICE,
       "stage1_s": round(t1, 4), "stage2_and_readjust_s": round(t12 - t1, 4), "stage3_s": round(t123 - t12, 4),
       "total_s": round(t123, 4), "us_per_tuning_step": round(t1 / n1 * 1e6, 1),
       "us_per_sample_transition": round(t_sample * 1e6, 1),
       "ess_kernel_ms_per_slice": round(t_ess * 1e3, 3), "ess_slice_shape": [n3, SLICE, D],
       "ess_lags_evaluated": {"min": int(lag_np.min()), "median": float(np.median(lag_np)), "max": int(lag_np.max()),
                              "of": n3}}
print(json.dumps(res))
