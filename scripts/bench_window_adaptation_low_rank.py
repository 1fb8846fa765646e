"""Time per warm-up step of window_adaptation_low_rank against the shared diagonal window_adaptation, NUTS, one GPU.

The low-rank step is split into its parts, each timed with CUDA events over repeated calls from the same state:
  transition   one NUTS transition under the rank-k low-rank metric (bjx_nuts_step, step-synchronous like the run loop)
  fast update  bjx_lowrank_window_update on a fast-stage step (block statistics + dual averaging)
  fold         a retained slow step minus a fast step (the two windowed covariance folds of draws and gradients)
  solve        a window end minus a retained slow step (merge, sigma, scatters, two top-k solves, float64 finish, install)
and the two whole warm-ups are timed end to end over the same number of steps.

    python scripts/bench_window_adaptation_low_rank.py [--chains 32768] [--dim 512] [--rank 10] [--steps 100]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import blackjax_b200 as bj  # noqa: E402
from blackjax_b200 import _engine, targets as T  # noqa: E402
from blackjax_b200.adaptation import low_rank_adaptation as lra  # noqa: E402


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chains", type=int, default=32768)
    ap.add_argument("--dim", type=int, default=512)
    ap.add_argument("--rank", type=int, default=10)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    C, D, k, dev = a.chains, a.dim, a.rank, "cuda:0"
    tgt = T.DiagGaussian(np.exp(np.linspace(-1.0, 1.0, D)), mean=np.zeros(D))
    x0 = torch.from_numpy(np.random.default_rng(0).standard_normal((C, D)).astype(np.float32)).to(dev)
    key = bj.random.key(0, dev)

    # ---- parts of one low-rank warm-up step ----
    state = bj.nuts.init(x0, tgt)
    eng = _engine.get_engine(x0, tgt, max_tree_depth=10)
    lw = lra._LowRankWindow(eng, k)
    lw.install(0.5)
    kernel = bj.nuts.build_kernel()
    acc = torch.full((C,), 0.8, device=dev)
    for _ in range(3):   # a few windows so that the metric and the solver's warm start are in place
        for b in (5, 5, 7):
            lw.update(state.position, state.logdensity_grad, acc, b, 0.8, 1e-5, 2.0)
    metric = lw.final()[2]
    keys = bj.random.split(key, a.reps + 1)
    it = iter(range(10 ** 9))
    st = [state]

    def transition():
        s, _ = kernel(keys[next(it) % len(keys)], st[0], tgt, 0.2, metric, max_num_doublings=5)
        st[0] = s

    t_tr = timed(transition, a.reps)
    q, g = st[0].position, st[0].logdensity_grad
    t_fast = timed(lambda: lw.update(q, g, acc, 0, 0.8, 1e-5, 2.0), a.reps)
    t_slow = timed(lambda: lw.update(q, g, acc, 5, 0.8, 1e-5, 2.0), a.reps)
    t_end = timed(lambda: lw.update(q, g, acc, 7, 0.8, 1e-5, 2.0), a.reps)
    iters, resid, noconv = lw.diagnostics()

    # ---- whole warm-ups over the same steps ----
    def whole(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / a.steps, out

    t_diag, (res_d, _) = whole(lambda: bj.window_adaptation(bj.nuts, tgt, shared=True, max_num_doublings=5).run(
        key, x0, num_steps=a.steps))
    t_lr, (res_l, _) = whole(lambda: bj.window_adaptation_low_rank(bj.nuts, tgt, max_rank=k, max_num_doublings=5).run(
        key, x0, num_steps=a.steps))
    print(json.dumps({
        "chains": C, "dim": D, "rank": k, "gpu": torch.cuda.get_device_name(0),
        "transition_ms": round(t_tr, 3), "fast_update_ms": round(t_fast, 3),
        "fold_ms": round(t_slow - t_fast, 3), "window_end_solve_ms": round(t_end - t_slow, 3),
        "eigensolver_iterations": iters, "eigensolver_residual": resid, "eigensolver_not_converged": noconv,
        "warmup_steps": a.steps, "shared_diagonal_ms_per_step": round(t_diag, 3),
        "low_rank_ms_per_step": round(t_lr, 3),
        "step_size_diagonal": res_d.parameters["step_size"], "step_size_low_rank": res_l.parameters["step_size"],
    }))


if __name__ == "__main__":
    main()
