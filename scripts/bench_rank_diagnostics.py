"""Rank-normalised diagnostics: ms per call of bjx_rank_diagnostics (R-hat, bulk ESS and tail ESS together) against the
classic effective_sample_size + potential_scale_reduction on the same history, the kernel split (sort, scores and
statistics, indicators, R-hat, ESS) from torch.profiler in a run of its own, and the sort's pairs per second and bytes
moved against the H100 SXM's 3.35 TB/s.  Workloads [T, C, D]: [1000, 4096, 64] and [200, 32768, 256], standard normal
draws, under the default 2 GiB scratch budget and an 8 GiB one.
The card's name and power limit are read in the same call.  CUDA events around `reps` calls after a warm-up.
usage: python scripts/bench_rank_diagnostics.py [reps] [out_dir]"""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import blackjax_b200 as bj  # noqa: E402
from blackjax_b200 import _lib, targets as T  # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
out_dir = sys.argv[2] if len(sys.argv) > 2 else None
dev = "cuda:0"
SHAPES = [(1000, 4096, 64), (200, 32768, 256)]
BUDGETS = [1 << 31, 1 << 33]
HBM = 3.35e12
# bytes per pair and sort: key build (read 4, write 8), then per 8-bit pass the tile histogram (read 8) and the scatter
# (read 8, write 8)
SORT_BYTES_PER_PAIR = 12 + 4 * 24

assert torch.cuda.is_available(), "the benchmark needs a CUDA device"


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
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def dims_per_pass(T_, C, D, budget):
    need = lambda dc: int(_lib.lib().bjx_rank_diagnostics_scratch_bytes(T_, C, D, dc))  # noqa: E731
    lo, hi = 0, D
    while lo < hi:
        mid = lo + (hi - lo + 1) // 2
        lo, hi = (mid, hi) if need(mid) <= budget else (lo, mid - 1)
    return lo - lo % 32 if 32 <= lo < D else lo


GROUPS = {"sort": ("k_rank_keys", "k_rank_sort_tile", "k_rank_hist", "k_rank_scan", "k_rank_scatter"),
          "scores and statistics": ("k_rank_scores",), "indicators": ("k_rank_indicator",),
          "rhat": ("k_chain_moments", "k_pooled_colstats", "k_rhat_finish"),
          "ess": ("k_ess_chain_mean", "k_ess_autocov", "k_ess_finish")}


def kernel_split(fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    split = {g: 0.0 for g in GROUPS}
    split["other"] = 0.0
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
        g = next((g for g, names in GROUPS.items() if any(n in e.key for n in names)), "other")
        split[g] += us / 1000.0
    return {g: round(v, 3) for g, v in split.items()}


results = {"gpu": smi("name"), "power_limit_w": smi("power.limit"), "reps": reps, "workloads": []}
profile_mode = os.environ.get("BJX_BENCH_PROFILE") == "1"
for T_, C, D in SHAPES:
    x = torch.randn(T_, C, D, device=dev, generator=torch.Generator(dev).manual_seed(0))
    tgt = T.StdNormal(D)
    n = 2 * C * (T_ // 2)
    row = {"shape": [T_, C, D], "pooled_draws_per_dim": n}
    if profile_mode:
        row["kernel_ms"] = kernel_split(lambda: bj.diagnostics._rank_diagnostics(x, tgt, 1 << 33, rhat=True))
        pairs = 2 * n * D                                          # R-hat sorts the draws and the folded draws
        sort_s = row["kernel_ms"]["sort"] / 1000.0
        row["sort_pairs_per_s"] = pairs / sort_s
        row["sort_bytes_per_s"] = pairs * SORT_BYTES_PER_PAIR / sort_s
        row["sort_share_of_hbm"] = round(row["sort_bytes_per_s"] / HBM, 3)
        row["kernel_ms_all_three"] = kernel_split(lambda: [f(x, tgt, max_scratch_bytes=1 << 33)
                                                           for f in (bj.rhat, bj.ess_bulk, bj.ess_tail)])
    else:
        row["classic_ess_plus_psr_ms"] = round(timed(lambda: (bj.diagnostics.effective_sample_size(x, tgt),
                                                              bj.diagnostics.potential_scale_reduction(x, tgt))), 3)
        for budget in BUDGETS:
            eng = bj._engine.get_engine(x[0], tgt)
            dc = dims_per_pass(T_, C, D, budget)
            nbytes = int(_lib.lib().bjx_rank_diagnostics_scratch_bytes(T_, C, D, dc))
            scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            outs = [torch.empty(D, device=dev) for _ in range(3)]
            L = _lib.lib()

            def call(prob=0.9):
                _lib.check(L.bjx_rank_diagnostics(eng.h, _lib.ptr(x), T_, prob, *(_lib.ptr(o) for o in outs),
                                                  _lib.ptr(scratch), nbytes), eng.h)

            def sort_only():
                _lib.check(L.bjx_rank_normalize(eng.h, _lib.ptr(x), T_, 0, _lib.ptr(out_rn), _lib.ptr(scratch), nbytes),
                           eng.h)

            out_rn = torch.empty(T_ // 2, 2 * C, D, device=dev)
            ms = timed(call)
            rn_ms = timed(sort_only)
            row[f"budget_{budget >> 30}GiB"] = {"dims_per_pass": dc, "scratch_bytes": nbytes,
                                                "rank_diagnostics_ms": round(ms, 3),
                                                "rank_normalize_ms": round(rn_ms, 3)}
            del scratch
    results["workloads"].append(row)
    del x
    torch.cuda.empty_cache()

print(json.dumps(results))
if out_dir:
    os.makedirs(out_dir, exist_ok=True)
    name = "rank_profile.json" if profile_mode else "rank_bench.json"
    with open(os.path.join(out_dir, name), "w") as f:
        json.dump(results, f, indent=1)
