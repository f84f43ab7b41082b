"""Cost of a learning-rate schedule on bench.py's workloads (bf16, CUDA-graph steps, one GPU).

  C5 against C5 with an ExponentialSchedule(ITERATION, lr, 0.9999) on every layer of G and D, and C2 against C2 with the same:
  1. Step time, `--rounds` alternating runs of `--steps` steps per configuration (CUDA events per step, L2 flushed between steps, as bench.py
     times its configurations), and the kernel launches per step.
  2. The updater kernels inside each step, timed with torch.profiler (CUDA activities) over 50 replayed steps in a separate run per
     configuration: the scheduled instantiation evaluates the schedule once per 4096-parameter block (thread 0, in double) and shares it
     through shared memory; everything else is the unscheduled kernel's pass.
The card's name, power limit and SM clock limit are read in the same process as the timings.
Usage: python tools/schedule_bench.py [--steps 100] [--rounds 3] [--out OUT.json]"""
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

CASES = (("c5", False), ("c5", True), ("c2", False), ("c2", True))
LAUNCH_STEPS = 5


def make(ctx, cfg_name, scheduled):
    cfg = bench.CONFIGS[cfg_name]
    G, D, gan = bench.make_gan(b, ctx, cfg, cfg["batch"])
    if scheduled:
        for net in (G, D):
            lr = net.learning_rate(next(s["name"] for s in net.specs if s.get("updater")))
            net.set_lr_schedule(models.exponential_schedule(lr, 0.9999))
    gan.upload(*bench.synthetic(cfg, cfg["batch"], 666))
    return cfg["batch"], G, D, gan


def name(cfg_name, scheduled):
    return cfg_name + ("+exponential_schedule" if scheduled else "")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except Exception as e:
        gpu = str(e)
    ctx = b.Context(0)
    res = {"gpu": gpu, "steps": args.steps, "runs": [], "updater_kernels": {}}
    for r in range(args.rounds):
        for cfg_name, scheduled in CASES:
            n, G, D, gan = make(ctx, cfg_name, scheduled)
            ms = bench.timed_resident_steps(ctx, gan, n, args.steps, 10, ctx.sync)
            l0 = ctx.launch_count()          # launches of graph-replayed steps only, counted around steps of their own
            for _ in range(LAUNCH_STEPS):
                gan.step_resident(n)
            ctx.sync()
            launches = (ctx.launch_count() - l0) / LAUNCH_STEPS
            res["runs"].append({"config": name(cfg_name, scheduled), "round": r, "ms_per_step": sum(ms) / len(ms), "samples_per_s": n * len(ms) / (sum(ms) * 1e-3),
                                "launches_per_step": launches})
            gan.close(); G.close(); D.close()
    for cfg_name, scheduled in CASES:
        n, G, D, gan = make(ctx, cfg_name, scheduled)
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
        res["updater_kernels"][name(cfg_name, scheduled)] = {"launches_per_step": len(t) / steps, "us_per_step": sum(t) / steps,
                                                            "params_G_plus_D": G.num_params() + D.num_params()}
        gan.close(); G.close(); D.close()
    ctx.close()
    print(json.dumps(res))
    if args.out:
        json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
