"""Cost of DL4J's L2 gradient normalization on bench.py's workloads (bf16, CUDA-graph steps, one GPU).

  C5 against C5 with RenormalizeL2PerLayer on G and D, and C2 against C2 with ClipL2PerLayer (threshold 1.0) on G and D:
  1. Step time, `--rounds` alternating runs of `--steps` steps per configuration (CUDA events per step, L2 flushed between steps, as bench.py
     times its configurations), and the kernel launches per step.
  2. The norm kernel inside each normalized step, timed with torch.profiler (CUDA activities) over 50 replayed steps in a separate run, and
     its achieved bandwidth against the H100 SXM data-sheet 3.35 TB/s.  Algorithmic bytes: the kernel reads every gradient once, 4 B per
     parameter of G and D per step (it writes one double per 4096 parameters and one float per parameter tensor).
The card's name, power limit and SM clock limit are read in the same process as the timings.
Usage: python tools/gradnorm_bench.py [--steps 100] [--rounds 3] [--out OUT.json]"""
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

CASES = (("c5", None, 1.0), ("c5", "renormalize_l2_per_layer", 1.0), ("c2", None, 1.0), ("c2", "clip_l2_per_layer", 1.0))


def make(ctx, cfg_name, mode, thr):
    cfg = bench.CONFIGS[cfg_name]
    G, D, gan = bench.make_gan(b, ctx, cfg, cfg["batch"])
    if mode:
        G.set_gradient_normalization(mode, thr); D.set_gradient_normalization(mode, thr)
    gan.upload(*bench.synthetic(cfg, cfg["batch"], 666))
    return cfg["batch"], G, D, gan


def name(cfg_name, mode):
    return cfg_name + ("+" + mode if mode else "")


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
    res = {"gpu": gpu, "steps": args.steps, "runs": [], "norm_kernel": {}}
    for r in range(args.rounds):
        for cfg_name, mode, thr in CASES:
            n, G, D, gan = make(ctx, cfg_name, mode, thr)
            l0 = ctx.launch_count()
            ms = bench.timed_resident_steps(ctx, gan, n, args.steps, 10, ctx.sync)
            launches = (ctx.launch_count() - l0) / (args.steps + max(3, 10))
            res["runs"].append({"config": name(cfg_name, mode), "round": r, "ms_per_step": sum(ms) / len(ms), "samples_per_s": n * len(ms) / (sum(ms) * 1e-3),
                                "launches_per_step": launches})
            gan.close(); G.close(); D.close()
    for cfg_name, mode, thr in CASES:
        if not mode:
            continue
        n, G, D, gan = make(ctx, cfg_name, mode, thr)
        params = G.num_params() + D.num_params()
        for _ in range(10):
            gan.step_resident(n)
        ctx.sync()
        steps = 50
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                gan.step_resident(n)
            ctx.sync()
        t = [ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
             for ev in prof.events() if "gradnorm_kernel" in ev.name and ev.device_type == torch.autograd.DeviceType.CUDA]
        us = sum(t) / steps
        byts = 4 * params
        gbs = byts / (us * 1e-6) / 1e9 if us > 0 else 0.0
        res["norm_kernel"][name(cfg_name, mode)] = {"launches_per_step": len(t) / steps, "us_per_step": us, "params_G_plus_D": params,
                                                    "algorithmic_MB_per_step": byts / 1e6, "achieved_GBps": gbs, "frac_of_3350_GBps": gbs / 3350.0}
        gan.close(); G.close(); D.close()
    ctx.close()
    print(json.dumps(res))
    if args.out:
        json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
