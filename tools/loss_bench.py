"""Cost of the discriminator's loss on bench.py's workloads (bf16, CUDA-graph steps, one GPU), and of the loss kernel on a regression output.

  C5 and C2 with D on XENT (what bench.py runs) and then on MSE (least-squares GAN labels 1 / 0 / 1), Hinge and Wasserstein (labels +1 / -1 / +1):
  1. Step time, `--rounds` alternating runs of `--steps` steps per configuration (CUDA events per step, L2 flushed between steps, as bench.py
     times its configurations), and the kernel launches per step.
  2. The loss kernels inside each step (xent_kernel or loss_kernel, two per step), timed with torch.profiler (CUDA activities) over 50 replayed
     steps in a separate run per configuration.
  3. The loss kernel alone on a [8192 x 256] MSE fit output (b2g_test_ew, bf16, identity and tanh) under torch.profiler, and the bytes per second
     it reaches at 8 B per element (z and dz 2 B each, the fp32 labels 4 B) as a fraction of the H100 SXM's 3.35 TB/s.  The operands were just
     uploaded, so part of them may come from L2: the fraction is an upper bound on the HBM rate, not a roofline.
The card's name, power limit and SM clock limit are read in the same process as the timings.
Usage: python tools/loss_bench.py [--steps 100] [--rounds 3] [--out OUT.json]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

import bench
import gan_deeplearning4j_b200 as b
from gan_deeplearning4j_b200 import models

LOSSES = ("xent", "mse", "hinge", "wasserstein")
HBM_BYTES_PER_S = 3.35e12
LAUNCH_STEPS = 5


def cuda_us(prof, name):
    return [ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            for ev in prof.events() if name in ev.name and ev.device_type == torch.autograd.DeviceType.CUDA]


def make(ctx, cfg_name, loss):
    cfg = bench.CONFIGS[cfg_name]
    gs, ds, gin, din = bench.build_specs(cfg)
    if loss != "xent":
        ds = models.mlp_discriminator(cfg["d"], cfg["hidden"], loss=loss) if cfg.get("mlp") else \
            models.dcgan_discriminator(cfg["size"], cfg["nf"], cfg["nc"], loss=loss)
    n = cfg["batch"]
    G = b.Net(ctx, gs, gin, max_batch=n, precision=b.BF16, xent_clip_eps=0.0, seed=666)
    D = b.Net(ctx, ds, din, max_batch=2 * n, precision=b.BF16, xent_clip_eps=0.0, bn_groups=2, seed=667)
    gan = b.Gan(G, D, fake_bn_train=False, use_cuda_graph=True)
    data = bench.synthetic(cfg, n, 666)
    if loss != "xent":
        lab = (1.0, 0.0, 1.0) if loss == "mse" else (1.0, -1.0, 1.0)
        data = data[:3] + [np.full((n, 1), v, np.float32) for v in lab]
    gan.upload(*data)
    return n, G, D, gan


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--configs", default="c5,c2")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    cases = [(c, k) for c in args.configs.split(",") for k in LOSSES]
    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except Exception as e:
        gpu = str(e)
    ctx = b.Context(0)
    res = {"gpu": gpu, "steps": args.steps, "runs": [], "loss_kernels": {}, "fit_output": {}}
    for r in range(args.rounds):
        for cfg_name, loss in cases:
            n, G, D, gan = make(ctx, cfg_name, loss)
            ms = bench.timed_resident_steps(ctx, gan, n, args.steps, 10, ctx.sync)
            l0 = ctx.launch_count()          # launches of graph-replayed steps only, counted around steps of their own
            for _ in range(LAUNCH_STEPS):
                gan.step_resident(n)
            ctx.sync()
            launches = (ctx.launch_count() - l0) / LAUNCH_STEPS
            res["runs"].append({"config": f"{cfg_name}+{loss}", "round": r, "ms_per_step": sum(ms) / len(ms), "samples_per_s": n * len(ms) / (sum(ms) * 1e-3),
                                "launches_per_step": launches, "losses": [float(v) for v in gan.losses()]})
            gan.close(); G.close(); D.close()
    for cfg_name, loss in cases:
        n, G, D, gan = make(ctx, cfg_name, loss)
        for _ in range(10):
            gan.step_resident(n)
        ctx.sync()
        steps = 50
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                gan.step_resident(n)
            ctx.sync()
        t = cuda_us(prof, "xent_kernel" if loss == "xent" else "loss_kernel")
        res["loss_kernels"][f"{cfg_name}+{loss}"] = {"launches_per_step": len(t) / steps, "us_per_step": sum(t) / steps}
        gan.close(); G.close(); D.close()
    rows, n_out, reps = 8192, 256, 50
    rng = np.random.default_rng(0)
    z = rng.standard_normal((rows, n_out)).astype(np.float32); y = rng.uniform(-1, 1, (rows, n_out)).astype(np.float32)
    for act in ("identity", "tanh"):
        call = lambda: b.test_ew(ctx, b.BF16, "loss", z, y, (z.size, 1, 0), act=act, loss="mse", rows=rows, cols=n_out, groups=1)
        call()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                call()
        t = cuda_us(prof, "loss_kernel")
        us = sum(t) / len(t)
        bytes_ = rows * n_out * 8
        res["fit_output"][f"mse+{act}"] = {"shape": [rows, n_out], "launches": len(t), "us_per_launch": us, "bytes": bytes_,
                                           "bytes_per_s": bytes_ / (us * 1e-6), "fraction_of_3_35_TBps": bytes_ / (us * 1e-6) / HBM_BYTES_PER_S}
    ctx.close()
    print(json.dumps(res))
    if args.out:
        json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
