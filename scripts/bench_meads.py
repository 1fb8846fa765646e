"""MEADS warm-up: time per warm-up step (fold statistics + one GHMC transition of every chain + the shuffle every K steps).
usage: python scripts/bench_meads.py [C] [D] [K] [steps] [rank]

With a rank (MEADS-LRD, e.g. `32768 512 4 200 16`), the diagonal and the low-rank runs alternate (two of each), then one
more low-rank run of the same steps is traced with torch.profiler to split the device time into statistics, the SYRK fold
of the covariance accumulator, the eigensolve and GHMC, and the eigensolver's iterations per solve are read from its
state.  The window starts at half the steps (the default fraction), so half the steps fold and solve."""
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import blackjax_b200 as bj

C = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
D = int(sys.argv[2]) if len(sys.argv) > 2 else 128
K = int(sys.argv[3]) if len(sys.argv) > 3 else 4
steps = int(sys.argv[4]) if len(sys.argv) > 4 else 200
rank = int(sys.argv[5]) if len(sys.argv) > 5 else None
dev = "cuda:0"
tgt = bj.targets.DiagGaussian(np.logspace(-1, 1, D))
q0 = bj.random.normal(bj.random.split(bj.random.key(7, dev), C), (D,))


def timed(warm, label):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    (last, params), _ = warm.run(bj.random.key(1, dev), q0, num_steps=steps)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    print(f"MEADS{label} C={C} D={D} K={K}: {ms / steps * 1e3:.1f} us per warm-up step ({steps} steps, {ms:.1f} ms); "
          f"step_size {float(params['step_size']):.4f} alpha {float(params['alpha']):.4f}")
    return params


if rank is None:
    warm = bj.meads_adaptation(tgt, num_chains=C, num_folds=K)
    warm.run(bj.random.key(0, dev), q0, num_steps=8)
    torch.cuda.synchronize()
    for rep in range(2):
        timed(warm, "")
    sys.exit(0)

try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
except OSError:
    q = "nvidia-smi unavailable"
print(f"device: {torch.cuda.get_device_name(0)}; nvidia-smi name, power limit: {q}")
diag = bj.meads_adaptation(tgt, num_chains=C, num_folds=K)
lrd = bj.meads_adaptation(tgt, num_chains=C, num_folds=K, low_rank_rank=rank)
for w in (diag, lrd):
    w.run(bj.random.key(0, dev), q0, num_steps=8)
torch.cuda.synchronize()
for rep in range(2):
    timed(diag, " diagonal")
    timed(lrd, f" LRD k={rank}")

# one traced LRD run: device time per phase, and the eigensolver's iterations
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from blackjax_b200.adaptation import meads_adaptation as mm  # noqa: E402

PHASES = {"syrk fold": ("k_block_stats", "k_cov_syrk", "k_cov_mean_update", "k_cov_merge"), "eigensolve": ("k_lrd_eig",),
          "ghmc": ("ghmc",), "shuffle": ("k_perm", "k_bitonic", "k_gather")}
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    lrd.run(bj.random.key(1, dev), q0, num_steps=steps)
    torch.cuda.synchronize()
split = {"statistics": 0.0, **{k: 0.0 for k in PHASES}}
for ev in prof.key_averages():
    t = getattr(ev, "device_time_total", None)
    if t is None:
        t = ev.cuda_time_total
    if t <= 0:
        continue
    name = ev.key
    phase = next((p for p, keys in PHASES.items() if any(k in name for k in keys)), "statistics")
    split[phase] += t
print("LRD device time per warm-up step (us, torch.profiler kernel times): " +
      ", ".join(f"{k} {v / steps:.1f}" for k, v in split.items()))

# iterations: the same run stepped by hand so that the eigensolver's state can be read
eng = mm._engine_for(q0, tgt)
lr = mm._LowRank(eng, min(rank, D), K)
lr.install()
folds = mm._Folds(eng, K)
st = bj.ghmc.init(q0.clone(), tgt, bj.random.key(2, dev))
kernel = bj.ghmc.build_kernel(inplace=True)
keys = bj.random.split(bj.random.key(3, dev), steps)
n = C // K
for t in range(steps):
    lr.update(folds, st.position, st.logdensity_grad, t, t >= steps // 2, 0.5, 1.0)
    st, _ = kernel(keys[t], st, tgt, None, None, None, None,
                   _rows=(folds.step_size, folds.alpha, folds.delta, None, None, n, ((t % K) * n, (t % K + 1) * n)))
h = lr.header.cpu().numpy()
solves = max(h[lr.SOLVES], 1)
print(f"eigensolver: {int(h[lr.SOLVES])} solves, mean {h[lr.ITERS_SUM] / solves:.1f} / max {int(h[lr.ITERS_MAX])} "
      f"iterations per solve, last residual {h[lr.RESID]:.2e} of max|mu|, non-converged flag {int(h[lr.NOCONV])}, "
      f"metric engaged {int(h[lr.ENGAGED])}")
