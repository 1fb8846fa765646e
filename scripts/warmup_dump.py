"""Window-adaptation outputs for comparing two builds byte for byte: runs, from seeded inputs on DiagGaussian targets,
* the shared diagonal window_adaptation with NUTS and with HMC at D = 24 and 512,
* window_adaptation_low_rank (rank 10) at D = 16 (D <= 2k: no eigensolver) and D = 64, NUTS and HMC, under Stan's schedule
  and the growing one,
* the per-chain window_adaptation with NUTS at D = 24,
and saves every run's per-step step sizes (the pooled recipes), final step size, metric and final positions to one .npz.
The default 4608 chains make the second statistic block ragged; 150 steps end at least one slow window under every schedule.
usage: python scripts/warmup_dump.py out.npz [C] [steps]"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import blackjax_b200 as bj  # noqa: E402
from blackjax_b200.adaptation.low_rank_adaptation import build_growing_window_schedule  # noqa: E402

out_path = sys.argv[1]
C = int(sys.argv[2]) if len(sys.argv) > 2 else 4608
steps = int(sys.argv[3]) if len(sys.argv) > 3 else 150
dev = "cuda:0"
ALGORITHMS = {"nuts": (bj.nuts, dict(max_num_doublings=5)), "hmc": (bj.hmc, dict(num_integration_steps=8))}
key = bj.random.key(11, dev)
out = {}


def setup(D):
    tgt = bj.targets.DiagGaussian(np.logspace(-1, 1, D))
    return tgt, bj.random.normal(bj.random.split(bj.random.key(7, dev), C), (D,))


def save(prefix, results, **arrays):
    out[prefix + "position"] = results.state.position.cpu().numpy()
    for name, a in arrays.items():
        out[prefix + name] = a.cpu().numpy() if hasattr(a, "cpu") else np.float32(a)
    print(prefix, "step size", np.asarray(out[prefix + "step_size"]).ravel()[:3], flush=True)


for D in (24, 512):
    tgt, q0 = setup(D)
    for name, (alg, extra) in ALGORITHMS.items():
        res, eps_hist = bj.window_adaptation(alg, tgt, shared=True, **extra).run(key, q0.clone(), num_steps=steps)
        save(f"shared_D{D}_{name}_", res, eps_history=eps_hist, step_size=res.parameters["step_size"],
             imm=res.parameters["inverse_mass_matrix"])

for D in (16, 64):
    tgt, q0 = setup(D)
    for name, (alg, extra) in ALGORITHMS.items():
        for sched, kw in (("stan", {}), ("growing", dict(schedule_fn=build_growing_window_schedule))):
            res, info = bj.window_adaptation_low_rank(alg, tgt, max_rank=10, **kw, **extra).run(key, q0.clone(), num_steps=steps)
            sigma, U, lam = res.parameters["inverse_mass_matrix"]
            save(f"low_rank_D{D}_{name}_{sched}_", res, eps_history=info.step_size, step_size=res.parameters["step_size"],
                 sigma=sigma, U=U, lam=lam, mu_star=info.mu_star, last_position=info.state.position)

tgt, q0 = setup(24)
res, _ = bj.window_adaptation(bj.nuts, tgt, max_num_doublings=5).run(key, q0.clone(), num_steps=steps)
save("per_chain_D24_nuts_", res, step_size=res.parameters["step_size"], imm=res.parameters["inverse_mass_matrix"])
np.savez(out_path, **out)
