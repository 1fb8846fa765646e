"""ChEES warm-up outputs for comparing two builds byte for byte: runs chees_adaptation(...).run with
mass_matrix_estimation=None and "diagonal" (plus the diagonal mode without the whitened criterion, without the length floor,
and with a window that never opens) on DiagGaussian targets of dimension 24, 200 and 1024, and saves every run's per-step
history, lambda_max and engaged flags, inverse mass matrix, step size, step count and final positions to one .npz.
The default 4608 chains make the second statistic block ragged; 100 steps open the window at step 50 and recompute the
slow-direction eigenvalue at steps 64 and 96.
usage: python scripts/chees_dump.py out.npz [C] [steps]"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import blackjax_b200 as bj  # noqa: E402
from blackjax_b200.adaptation.chees_adaptation import adam  # noqa: E402

out_path = sys.argv[1]
C = int(sys.argv[2]) if len(sys.argv) > 2 else 4608
steps = int(sys.argv[3]) if len(sys.argv) > 3 else 100
dev = "cuda:0"
DIAG = dict(mass_matrix_estimation="diagonal")
CONFIGS = {"none": {}, "diagonal": DIAG, "diagonal_unwhitened": dict(DIAG, _whiten_criterion=False),
           "diagonal_no_floor": dict(DIAG, _length_floor=False), "diagonal_window_1": dict(DIAG, mass_matrix_window_fraction=1.0)}

out = {}
for D in (24, 200, 1024):
    tgt = bj.targets.DiagGaussian(np.logspace(-1, 1, D))
    q0 = bj.random.normal(bj.random.split(bj.random.key(7, dev), C), (D,))
    for name, kw in CONFIGS.items():
        warm = bj.chees_adaptation(tgt, num_chains=C, **kw)
        (state, params), info = warm.run(bj.random.key(11, dev), q0.clone(), step_size=0.05, optim=adam(0.05), num_steps=steps)
        p = f"D{D}_{name}_"
        if kw:
            out[p + "history"] = info.history.numpy()
            out[p + "lambda_max"] = info.lambda_max.numpy()
            out[p + "engaged"] = info.engaged.numpy()
            out[p + "floor_clipped_by_cap"] = np.bool_(info.floor_clipped_by_cap)
        else:
            out[p + "history"] = info.numpy()
        out[p + "imm"] = params["inverse_mass_matrix"].cpu().numpy()
        out[p + "step_size"] = np.float32(params["step_size"])
        out[p + "n_lf"] = np.float32(params["integration_steps_params"][0])
        out[p + "position"] = state.position.cpu().numpy()
        print(f"D={D} {name}: step size {params['step_size']:.5f}, n_lf {params['integration_steps_params'][0]:.3f}", flush=True)
np.savez(out_path, **out)
