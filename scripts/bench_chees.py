"""ChEES warm-up: time per warm-up step with mass_matrix_estimation=None and "diagonal" (alternated in one process), and
the windowed covariance accumulator's SYRK (k_cov_syrk + its mean update) on its own: CUDA-event time and achieved FP32
FLOP/s (C * D * (D + 1) per fold) against the H100 SXM data sheet's 67 TFLOP/s.
usage: python scripts/bench_chees.py [C] [D] [steps]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import blackjax_b200 as bj
from blackjax_b200 import _engine
from blackjax_b200._lib import CHEES_LENGTH_FLOOR, CHEES_WHITEN, check, lib, ptr
from blackjax_b200.adaptation.chees_adaptation import adam

C = int(sys.argv[1]) if len(sys.argv) > 1 else 32768
D = int(sys.argv[2]) if len(sys.argv) > 2 else 512
steps = int(sys.argv[3]) if len(sys.argv) > 3 else 100
dev = "cuda:0"
PEAK_FP32 = 67e12


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        pl = "unknown"
    return name, pl


tgt = bj.targets.DiagGaussian(np.logspace(-1, 1, D))
q0 = bj.random.normal(bj.random.split(bj.random.key(7, dev), C), (D,))
modes = {"None": bj.chees_adaptation(tgt, num_chains=C),
         "diagonal": bj.chees_adaptation(tgt, num_chains=C, mass_matrix_estimation="diagonal")}
for w in modes.values():  # warm-up: compile caches, allocations
    w.run(bj.random.key(0, dev), q0, step_size=0.05, optim=adam(0.05), num_steps=4)
torch.cuda.synchronize()
times = {k: [] for k in modes}
for rep in range(3):
    for k, w in modes.items():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        (last, params), _ = w.run(bj.random.key(1, dev), q0, step_size=0.05, optim=adam(0.05), num_steps=steps)
        e1.record()
        torch.cuda.synchronize()
        times[k].append(e0.elapsed_time(e1) / steps * 1e3)

# the SYRK fold on its own
opts = CHEES_WHITEN | CHEES_LENGTH_FLOOR
eng = _engine.get_engine(q0, tgt)
L_ = lib()
ms = torch.empty(L_.bjx_chees_metric_state_floats(C, D, 1, opts), device=dev)
imm = torch.empty(D, device=dev)
check(L_.bjx_chees_metric_init(eng.h, ptr(ms), 1, opts, ptr(imm)), eng.h)
for _ in range(3):
    check(L_.bjx_chees_metric_fold_covariance(eng.h, opts, ptr(ms), ptr(q0)), eng.h)
check(L_.bjx_synchronize(eng.h), eng.h)
torch.cuda.synchronize()
reps = 20
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(reps):
    check(L_.bjx_chees_metric_fold_covariance(eng.h, opts, ptr(ms), ptr(q0)), eng.h)
check(L_.bjx_synchronize(eng.h), eng.h)
e1.record()
torch.cuda.synchronize()
fold_us = e0.elapsed_time(e1) / reps * 1e3
flop = C * D * (D + 1)
name, pl = card()
res = {"card": name, "power_limit": pl, "C": C, "D": D, "steps": steps,
       "us_per_step_none": round(float(np.median(times["None"])), 1),
       "us_per_step_diagonal": round(float(np.median(times["diagonal"])), 1),
       "syrk_fold_us": round(fold_us, 1), "syrk_tflops": round(flop / fold_us * 1e-6, 2),
       "syrk_fraction_of_fp32_peak": round(flop / (fold_us * 1e-6) / PEAK_FP32, 3)}
print(f"ChEES C={C} D={D} on {name} ({pl}): None {res['us_per_step_none']} us/step, diagonal "
      f"{res['us_per_step_diagonal']} us/step; SYRK fold {fold_us:.1f} us = {res['syrk_tflops']} TFLOP/s "
      f"({100 * res['syrk_fraction_of_fp32_peak']:.1f} % of 67 TFLOP/s)")
print(json.dumps(res))
