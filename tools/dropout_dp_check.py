"""Two-rank DropoutLayer check, run under torchrun:  python -m torch.distributed.run --nproc-per-node 2 tools/dropout_dp_check.py OUT.json
Every rank trains the same MLP-GAN with DropoutLayers in D on identical data (CUDA graph replay, gradient all-reduce).  The rank enters each
mask's counter, so the ranks draw different masks, while the all-reduced gradients keep D's parameters identical across ranks.  Rank 0
writes the results to OUT.json; tests/test_gpu_dropout.py runs it when the machine has >= 2 GPUs."""
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
from oracle.dl4j_oracle import dropout_mask  # noqa: E402  (the oracle's NumPy restatement of the mask)

rank, world, local = parallel.env_rank_world()
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
ctx = b.Context(local)
parallel.attach_communicator(ctx, dist, rank, world)
n, z, hid, d = 128, 128, 256, 128
G = b.Net(ctx, m.mlp_generator(z, hid, d, lr=1e-3), (z,), max_batch=n, precision=b.BF16, xent_clip_eps=0.0, seed=1)
ds = m.mlp_discriminator(d, hid, lr=1e-3, dropout=0.5)
D = b.Net(ctx, ds, (d,), max_batch=2 * n, precision=b.BF16, xent_clip_eps=0.0, bn_groups=2, seed=2)
gan = b.Gan(G, D, use_cuda_graph=True)
rng = np.random.default_rng(7)          # the same data on every rank
data = [rng.uniform(-1, 1, (n, d)), rng.uniform(-1, 1, (n, z)), rng.uniform(-1, 1, (n, z)),
        1 + 0.05 * rng.standard_normal((n, 1)), 0.05 * rng.standard_normal((n, 1)), np.ones((n, 1))]
for _ in range(3):
    gan.step(*data)
li = [i for i, s in enumerate(ds) if s["type"] == "dropout"][0]
act = D.activation(li, n)                 # the generator step's D pass of step 3: pass 5
mask_ok = bool(np.array_equal(act.reshape(n, hid) != 0, dropout_mask(2, rank, li, 5, n, 1, 1, hid, 0.5).reshape(n, hid)))
mine = torch.tensor(np.concatenate([D.params(), act.ravel()]), device=f"cuda:{local}")
allv = [torch.empty_like(mine) for _ in range(world)]
dist.all_gather(allv, mine)
allv = [t.cpu().numpy() for t in allv]
npar = D.num_params()
ok = torch.tensor([1.0 if mask_ok else 0.0], device=f"cuda:{local}")
dist.all_reduce(ok, op=dist.ReduceOp.MIN)
if rank == 0:
    res = {"world": world, "d_params_identical": all(np.array_equal(allv[0][:npar], v[:npar]) for v in allv[1:]),
           "dropout_activations_differ": all(not np.array_equal(allv[0][npar:], v[npar:]) for v in allv[1:]), "masks_match_oracle": bool(ok.item() == 1.0)}
    json.dump(res, open(sys.argv[1], "w"))
    print(json.dumps(res))
gan.close(); G.close(); D.close(); ctx.close()
dist.destroy_process_group()
