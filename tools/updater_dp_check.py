"""Two-rank parameter averaging of the three-slot updater state, run under torchrun:
    python -m torch.distributed.run --nproc-per-node 2 tools/updater_dp_check.py OUT.json
Every rank fits its own copy of an FP32 MLP whose layers use AMSGrad (three state slots), Nadam and AdaGrad on its own data with the gradient
all-reduce switched off (ParameterAveragingTrainingMaster mode), then b2g_net_average_parameters averages the parameters and every state slot
on the device.  Rank 0 checks the result against the mean of what the ranks held before and writes it to OUT.json;
tests/test_gpu_updaters.py runs it when the machine has >= 2 GPUs."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import torch.distributed as dist

import gan_deeplearning4j_b200 as b
from gan_deeplearning4j_b200 import models as m, parallel

rank, world, local = parallel.env_rank_world()
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
ctx = b.Context(local)
parallel.attach_communicator(ctx, dist, rank, world)
specs = [{"type": "dense", "name": "d1", "n_out": 96, "activation": "tanh", "updater": m.amsgrad(2e-3)},
         {"type": "dense", "name": "d2", "n_out": 64, "activation": "lrelu", "alpha": 0.2, "updater": m.nadam(1e-3)},
         {"type": "output", "name": "out", "n_out": 1, "updater": m.adagrad(0.02)}]
net = b.Net(ctx, specs, (40,), max_batch=16, precision=b.FP32, seed=3)
net.set_grad_allreduce(False)
rng = np.random.default_rng(100 + rank)           # different data on every rank
for _ in range(3):
    net.fit(rng.uniform(-1, 1, (16, 40)), rng.uniform(0, 1, (16, 1)))
before = np.concatenate([net.params(), net.updater_state()]).astype(np.float64)
t = torch.tensor(before, device=f"cuda:{local}")
allv = [torch.empty_like(t) for _ in range(world)]
dist.all_gather(allv, t)
want = sum(v.cpu().numpy() for v in allv) / world
net.average_parameters()
after = np.concatenate([net.params(), net.updater_state()]).astype(np.float64)
n = net.num_params()
if rank == 0:
    err = np.abs(after - want) / (np.abs(want) + 1e-30)
    res = {"world": world, "state_slots": int(net.updater_state_size() // n), "ranks_differed": bool(np.abs(allv[0].cpu().numpy() - allv[-1].cpu().numpy()).max() > 0),
           "max_rel_err_params": float(err[:n].max()), "max_rel_err_slot": [float(err[n * (k + 1):n * (k + 2)].max()) for k in range(3)]}
    json.dump(res, open(sys.argv[1], "w"))
    print(json.dumps(res))
net.close()
ctx.close()
dist.destroy_process_group()
