"""Worker of tests/test_gpu_chees_metric.py::test_chees_diagonal_bit_identical_on_one_and_two_gpus: ChEES with
mass_matrix_estimation="diagonal" over C_total = chains_per_rank x world chains, sharded over `world` GPUs; rank 0 saves
the histories, the adapted parameters and every chain's final position in global chain order.
usage: [torchrun ...] chees_metric_worker.py out.npz chains_per_rank"""
import os
import sys

import numpy as np
import torch

import blackjax_b200 as bj
from blackjax_b200.adaptation.chees_adaptation import adam

out, C = sys.argv[1], int(sys.argv[2])
world, rank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0"))
local = int(os.environ.get("LOCAL_RANK", "0"))
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
if world > 1:
    import torch.distributed as dist
    dist.init_process_group("nccl", device_id=dev)
D, T_ = 48, 80
tgt = bj.targets.DiagGaussian(np.logspace(-1, 1, D))
q0 = bj.random.normal(bj.random.split(bj.random.key(7, dev), C * world)[rank * C:(rank + 1) * C], (D,))
warm = bj.chees_adaptation(tgt, num_chains=C, mass_matrix_estimation="diagonal", mass_matrix_window_fraction=0.2)
(state, params), info = warm.run(bj.random.key(11, dev), q0, step_size=0.05, optim=adam(0.05), num_steps=T_)
pos = state.position
if world > 1:
    allp = [torch.empty_like(pos) for _ in range(world)]
    dist.all_gather(allp, pos)
    pos = torch.cat(allp)
if rank == 0:
    np.savez(out, n_ranks=world, history=info.history.numpy(), lambda_max=info.lambda_max.numpy(),
             engaged=info.engaged.numpy(), imm=params["inverse_mass_matrix"].cpu().numpy(),
             step_size=np.float32(params["step_size"]), n_lf=np.float32(params["integration_steps_params"][0]),
             position=pos.cpu().numpy())
if world > 1:
    dist.barrier()
    dist.destroy_process_group()
