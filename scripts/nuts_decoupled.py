"""Decoupled-chains NUTS sampler (bjx_nuts_sample / k_nuts_chains) vs T calls of the step kernel (nuts.step with the keys
split(rng_key, T)): same draws, time per transition.  usage: python scripts/nuts_decoupled.py [C] [D] [T]"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import blackjax_b200 as bj

C = int(sys.argv[1]) if len(sys.argv) > 1 else 65536
D = int(sys.argv[2]) if len(sys.argv) > 2 else 128
T = int(sys.argv[3]) if len(sys.argv) > 3 else 64
dev = "cuda:0"
tgt = bj.targets.Funnel(D)
imm = torch.ones(D, device=dev)
q0 = 0.1 * bj.random.normal(bj.random.split(bj.random.key(7, dev), C), (D,))
st = bj.nuts.init(q0, tgt)
eps = 0.25
# burn in so that the trees have their stationary depth profile
st, _, _, _ = bj.sample_nuts_native(bj.random.key(1, dev), st, tgt, eps, imm, 40, keep_history=False)
torch.cuda.synchronize()
alg = bj.nuts(tgt, eps, imm, max_num_doublings=10)
key = bj.random.key(2, dev)


def decoupled():
    fin, _, _, n_int = bj.sample_nuts_native(key, st, tgt, eps, imm, T, keep_history=False)
    return fin, n_int.sum()


def stepwise():
    s, lf = st, 0
    for k in bj.random.split(key, T):
        s, info = alg.step(k, s)
        lf = lf + info.num_integration_steps.sum()
    return s, lf


for rep in range(3):
    for name, run in (("decoupled", decoupled), ("step kernel", stepwise)):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fin, lf = run()
        e1.record()
        torch.cuda.synchronize()
        ms, lf = e0.elapsed_time(e1), int(lf)
        print(f"{name} C={C} D={D} T={T}: {ms / T:.4f} ms/transition, {lf / ms * 1e3:.3e} leapfrogs/s, "
              f"mean tree {lf / (C * T):.2f}, checksum {float(fin.position.double().sum()):.9e} {lf}")
