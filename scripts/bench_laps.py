"""LAPS (blackjax_b200.adaptation.laps) on the diagonal Gaussian.  Reports, with the card's name, power limit and clocks
read in the same run, one JSON line per shape:
* the burn-in step (bjx_laps_burn_in_step, equi_full off and on) against one bjx_mclmc_sample transition (velocity Verlet,
  identity metric) on the same chains, from CUDA events over `reps` steps after a warm-up;
* the kernels of a burn-in step from torch.profiler in a run of their own: the fused transition k_laps_burn_in, the
  merge (k_laps_colsum), the update (k_laps_update) and the four equi_full kernels;
* the adjusted step (bjx_laps_adjusted_step, 15 steps, omelyan) against bjx_adjusted_mclmc_step on the same chains and step size;
* one whole laps() run (num_steps1, num_steps2 below, early stop on), from a host clock around a synchronised call.
usage: python scripts/bench_laps.py [C D [C D ...]]"""
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import blackjax_b200 as bj
from blackjax_b200 import _engine
from blackjax_b200._lib import check, lib, ptr
from blackjax_b200.adaptation import laps as L
from blackjax_b200.adaptation import laps_burn_in as lb
from blackjax_b200.mcmc import integrators

dev = "cuda:0"
args = [int(a) for a in sys.argv[1:]] or [65536, 1024, 4096, 100]
SHAPES = list(zip(args[0::2], args[1::2]))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = "unknown"
    return out


def events(fn, reps, warm=2):
    for _ in range(warm):
        fn(0)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(reps):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def kernel_ms(fn, reps):
    """mean device time per call of each kernel whose name contains one of the LAPS kernel names"""
    names = ("k_laps_burn_in", "k_laps_colsum", "k_laps_update", "k_laps_rademacher", "k_laps_zg<", "k_laps_zgx",
             "k_laps_equi_full")
    fn(0)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for i in range(reps):
            fn(i)
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for n in names:
            key = n.rstrip("<")
            if key in ev.key and (n != "k_laps_zg<" or "k_laps_zgx" not in ev.key):
                out[key] = out.get(key, 0.0) + ev.device_time_total / 1e3 / reps
    return out


def shape(C, D, reps):
    s = np.exp(np.linspace(0.0, np.log(3.0), D))
    tgt = bj.targets.DiagGaussian(s, mean=np.full(D, 1.0))
    q0 = bj.random.normal(bj.random.split(bj.random.key(7, dev), C), (D,))
    eng = _engine.get_engine(q0, tgt)
    eng.set_integrator(integrators.velocity_verlet)
    T = min(4096, (1 << 32) // C - 1)  # keys: chain index * T + t below 2^32
    res = {"chains": C, "dims": D}
    for equi in (False, True):
        adap = lb.new_state(eng, 20, equi)
        st = lb.initialize(eng, q0, adap, 20)
        cfg = lb.config(20, early_stop=False, equi_full=equi)
        key = np.array([1, 2], np.uint32)
        step = lambda i: lb.burn_in_step_(eng, key, i % T, T, st, adap, cfg)
        res["burn_in_step_ms" + ("_equi_full" if equi else "")] = events(step, reps)
        if equi:
            res["burn_in_kernels_ms"] = kernel_ms(step, reps)
            eps, Lv = lb.header(adap)["step_size"], lb.header(adap)["L"]
    # bjx_mclmc_sample at the burn-in's last (step size, L): one transition per step
    q, u, logp, g = (x.clone() for x in st)
    k = bj.random.key(3, dev)
    cutoff = math.inf

    def mclmc(i):
        check(lib().bjx_mclmc_sample(eng.h, ptr(k), ptr(q), ptr(u), ptr(logp), ptr(g), float(eps), None, float(Lv),
                                     None, cutoff, 1, None, 1, None), eng.h)
    res["mclmc_sample_step_ms"] = events(mclmc, reps)
    res["burn_in_eps_L"] = [eps, Lv]
    # adjusted phase, omelyan, 15 steps per sample, against bjx_adjusted_mclmc_step at the same step size and metric
    lb.switch_(eng, adap, True)
    eng.set_integrator(integrators.omelyan)
    S = T
    ast = (st[0], st[2], st[3])
    res["adjusted_step_ms"] = events(lambda i: lb.adjusted_step_(eng, key, i % S, S, ast, adap, 20, 15, 0.9, True), reps)
    keys = bj.random.split(bj.random.key(5, dev), C)
    e = lb.header(adap)["step_size"]
    out = tuple(torch.empty_like(x) for x in ast)
    res["adjusted_mclmc_step_ms"] = events(lambda i: eng.adjusted_mclmc_step(keys, *ast, e, 15, 1.25, out=out), reps)
    res["adjusted_step_size"] = e
    del adap, st, q, u, logp, g, out
    torch.cuda.empty_cache()
    # one whole run
    n1, n2 = 200, 2000
    L.laps(tgt, lambda kk: bj.random.normal(kk, (D,)), D, 20, 150, C, None, bj.random.key(1, dev))  # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    info, gcps, _, _ = L.laps(tgt, lambda kk: bj.random.normal(kk, (D,)), D, n1, n2, C, None, bj.random.key(1, dev))
    torch.cuda.synchronize()
    res["laps_run_s"] = time.perf_counter() - t0
    res["laps_run"] = {"num_steps1": n1, "num_steps2": n2, "burn_in_steps_run": len(info["phase_1"]["L"]),
                       "adjusted_steps": len(info["phase_2"]["L"]), "gradient_calls_per_step": gcps}
    return res


if __name__ == "__main__":
    print(json.dumps({"card": card()}), flush=True)
    for C, D in SHAPES:
        r = shape(C, D, reps=20)
        r["card_after"] = card()
        print(json.dumps(r), flush=True)
