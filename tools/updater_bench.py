"""Cost of the updater kinds on bench.py's workloads (bf16, CUDA-graph steps, one GPU).

  C5 and C2 with every layer of G and D on Adam (the baseline, what bench.py runs) and then on each of Nesterovs, AdaGrad, AdaMax, Nadam, AMSGrad
  and AdaDelta in turn:
  1. Step time, `--rounds` alternating runs of `--steps` steps per configuration (CUDA events per step, L2 flushed between steps, as bench.py
     times its configurations), and the kernel launches per step.
  2. The updater kernels inside each step, timed with torch.profiler (CUDA activities) over 50 replayed steps in a separate run per
     configuration, and the bytes per second they reach from the per-kind traffic (include/b200gan.h, DESIGN.md 3): Nesterovs and AdaGrad
     20 B/param, Adam, AdaMax, Nadam and AdaDelta 28 B, AMSGrad 36 B, each + 2 B for the bf16 operand copy, as a fraction of the H100 SXM's
     3.35 TB/s.  The gradients were written by the backward pass just before, so part of them comes from L2: the fraction is an upper bound
     on the HBM rate the kernel needs, not a roofline.
The card's name, power limit and SM clock limit are read in the same process as the timings.
Usage: python tools/updater_bench.py [--steps 100] [--rounds 3] [--out OUT.json]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

import bench
import gan_deeplearning4j_b200 as b
from gan_deeplearning4j_b200 import models

KINDS = ("adam", "nesterovs", "adagrad", "adamax", "nadam", "amsgrad", "adadelta")
BYTES_PER_PARAM = {"adam": 28, "nesterovs": 20, "adagrad": 20, "adamax": 28, "nadam": 28, "amsgrad": 36, "adadelta": 28}
HBM_BYTES_PER_S = 3.35e12
LAUNCH_STEPS = 5


def with_kind(specs, kind):
    """Every updater of the specs replaced by `kind` at the layer's Adam learning rate (AdaDelta: DL4J's defaults, no learning rate)."""
    out = []
    for s in specs:
        s = dict(s)
        if s.get("updater"):
            lr = s["updater"]["lr"]
            s["updater"] = models.adadelta() if kind == "adadelta" else models.nesterovs(lr) if kind == "nesterovs" else getattr(models, kind)(lr)
        out.append(s)
    return out


def make(ctx, cfg_name, kind):
    cfg = bench.CONFIGS[cfg_name]
    gs, ds, gin, din = bench.build_specs(cfg)
    n = cfg["batch"]
    G = b.Net(ctx, with_kind(gs, kind), gin, max_batch=n, precision=b.BF16, xent_clip_eps=0.0, seed=666)
    D = b.Net(ctx, with_kind(ds, kind), din, max_batch=2 * n, precision=b.BF16, xent_clip_eps=0.0, bn_groups=2, seed=667)
    gan = b.Gan(G, D, fake_bn_train=False, use_cuda_graph=True)
    gan.upload(*bench.synthetic(cfg, n, 666))
    return n, G, D, gan


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--configs", default="c5,c2")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    cases = [(c, k) for c in args.configs.split(",") for k in KINDS]
    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except Exception as e:
        gpu = str(e)
    ctx = b.Context(0)
    res = {"gpu": gpu, "steps": args.steps, "runs": [], "updater_kernels": {}}
    for r in range(args.rounds):
        for cfg_name, kind in cases:
            n, G, D, gan = make(ctx, cfg_name, kind)
            ms = bench.timed_resident_steps(ctx, gan, n, args.steps, 10, ctx.sync)
            l0 = ctx.launch_count()          # launches of graph-replayed steps only, counted around steps of their own
            for _ in range(LAUNCH_STEPS):
                gan.step_resident(n)
            ctx.sync()
            launches = (ctx.launch_count() - l0) / LAUNCH_STEPS
            res["runs"].append({"config": f"{cfg_name}+{kind}", "round": r, "ms_per_step": sum(ms) / len(ms), "samples_per_s": n * len(ms) / (sum(ms) * 1e-3),
                                "launches_per_step": launches})
            gan.close(); G.close(); D.close()
    for cfg_name, kind in cases:
        n, G, D, gan = make(ctx, cfg_name, kind)
        for _ in range(10):
            gan.step_resident(n)
        ctx.sync()
        steps = 50
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                gan.step_resident(n)
            ctx.sync()
        t = [ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
             for ev in prof.events() if "updater_kernel" in ev.name and ev.device_type == torch.autograd.DeviceType.CUDA]
        params = G.num_params() + D.num_params()
        us = sum(t) / steps
        bytes_ = params * (BYTES_PER_PARAM[kind] + 2)
        res["updater_kernels"][f"{cfg_name}+{kind}"] = {"launches_per_step": len(t) / steps, "us_per_step": us, "params_G_plus_D": params,
                                                       "bytes_per_step": bytes_, "bytes_per_s": bytes_ / (us * 1e-6) if us else None,
                                                       "fraction_of_3_35_TBps": bytes_ / (us * 1e-6) / HBM_BYTES_PER_S if us else None}
        gan.close(); G.close(); D.close()
    ctx.close()
    print(json.dumps(res))
    if args.out:
        json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
