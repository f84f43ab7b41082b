"""Two-rank weight-constraint check, run under torchrun:  python -m torch.distributed.run --nproc-per-node 2 tools/constraint_dp_check.py OUT.json
Every rank trains the same FP32 MLP-GAN on identical data (gradient all-reduce, CUDA graph replay after the first step) with MaxNorm on every
W: whole-tensor groups on G (one-pass and two-launch contiguous paths) and groups over nOut on D (dims {1}: strided groups, two launches).  The
constraints act on the all-reduced update, so the ranks end with identical parameters, and replicated data gives what one GPU computes on that
data alone.  Rank 0 writes the results to OUT.json; tests/test_gpu_constraints.py runs it when the machine has >= 2 GPUs."""
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
n, z, hid, d = 64, 32, 128, 48
rng = np.random.default_rng(7)          # the same data on every rank
data = [rng.uniform(-1, 1, (n, d)), rng.uniform(-1, 1, (n, z)), rng.uniform(-1, 1, (n, z)),
        1 + 0.05 * rng.standard_normal((n, 1)), 0.05 * rng.standard_normal((n, 1)), np.ones((n, 1))]


def train(ctx):
    G = b.Net(ctx, m.mlp_generator(z, hid, d, lr=1e-3), (z,), max_batch=n, precision=b.FP32, seed=1, constraints=[m.max_norm(2.0, ())])
    D = b.Net(ctx, m.mlp_discriminator(d, hid, lr=1e-3), (d,), max_batch=2 * n, precision=b.FP32, bn_groups=2, seed=2,
              constraints=[m.max_norm(0.5, (1,))])
    gan = b.Gan(G, D, use_cuda_graph=True)
    for _ in range(3):
        gan.step(*data)
    out = np.concatenate([G.params(), D.params()])
    gan.close(); G.close(); D.close()
    return out


single = train(b.Context(local))          # this GPU alone, no communicator
ctx = b.Context(local)
parallel.attach_communicator(ctx, dist, rank, world)
mine = train(ctx)
t = torch.tensor(mine, device=f"cuda:{local}")
allv = [torch.empty_like(t) for _ in range(world)]
dist.all_gather(allv, t)
allv = [v.cpu().numpy() for v in allv]
if rank == 0:
    res = {"world": world, "params_identical_across_ranks": all(np.array_equal(allv[0], v) for v in allv[1:]),
           "max_rel_err_vs_one_gpu": float(np.abs(mine - single).max() / np.abs(single).max()), "moved": float(np.abs(mine).max())}
    json.dump(res, open(sys.argv[1], "w"))
    print(json.dumps(res))
ctx.close()
dist.destroy_process_group()
