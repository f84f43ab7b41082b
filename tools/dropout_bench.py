"""DropoutLayer cost on the C5 workload (bench.py's MLP-GAN: d=256, z=128, hidden 1024-1024, bf16, batch 8192 per GPU).

C5D is C5 with DropoutLayer(0.5) after each hidden LeakyReLU of D, the shape of DL4J's MNIST GAN example discriminator.
  1. Step time of C5 and C5D, `--rounds` alternating runs of `--steps` CUDA-graph steps each (CUDA events per step, L2 flushed between
     steps, as bench.py times its configurations).
  2. The dropout kernels inside the C5D step, timed with torch.profiler (CUDA activities) over 50 replayed steps, and their achieved bandwidth
     against the H100 SXM data-sheet 3.35 TB/s.  Bytes per masked element, bf16: forward reads x (2 B), writes y (2 B) and one mask bit;
     backward reads dy (2 B) and the bit, writes dx (2 B).  Per step D runs them on its 2N-row pass and on the generator step's N-row pass,
     over two hidden layers.
Usage: python tools/dropout_bench.py [--steps 100] [--rounds 3] [--out OUT.json]"""
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
from gan_deeplearning4j_b200 import models as m

C5 = bench.CONFIGS["c5"]


def make(ctx, dropout):
    n = C5["batch"]
    G = b.Net(ctx, m.mlp_generator(C5["z"], C5["hidden"], C5["d"]), (C5["z"],), max_batch=n, precision=b.BF16, xent_clip_eps=0.0, seed=666)
    D = b.Net(ctx, m.mlp_discriminator(C5["d"], C5["hidden"], dropout=dropout), (C5["d"],), max_batch=2 * n, precision=b.BF16, xent_clip_eps=0.0,
              bn_groups=2, seed=667)
    gan = b.Gan(G, D, fake_bn_train=False, use_cuda_graph=True)
    gan.upload(*bench.synthetic(C5, n, 666))
    return G, D, gan


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    n, hid = C5["batch"], C5["hidden"]
    ctx = b.Context(0)
    res = {"workload": C5["desc"] + "; C5D: DropoutLayer(0.5) after each hidden LeakyReLU of D", "steps": args.steps, "runs": []}
    for r in range(args.rounds):
        for name, p in (("c5", None), ("c5d", 0.5)):
            G, D, gan = make(ctx, p)
            l0 = ctx.launch_count()
            ms = bench.timed_resident_steps(ctx, gan, n, args.steps, 10, ctx.sync)
            launches = (ctx.launch_count() - l0) / (args.steps + 10)
            res["runs"].append({"config": name, "round": r, "ms_per_step": sum(ms) / len(ms), "samples_per_s": n * len(ms) / (sum(ms) * 1e-3),
                                "launches_per_step": launches})
            gan.close(); G.close(); D.close()
    G, D, gan = make(ctx, 0.5)
    for _ in range(10):
        gan.step_resident(n)
    ctx.sync()
    steps = 50
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            gan.step_resident(n)
        ctx.sync()
    t = {"fwd": [], "bwd": []}
    for ev in prof.events():
        for k in t:
            if f"dropout_{k}_kernel" in ev.name and ev.device_type == torch.autograd.DeviceType.CUDA:
                t[k].append(ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total)
    elems = 2 * (2 * n + n) * hid                  # masked elements per step, forward (the backward handles the same)
    bytes_el = 2 + 2 + 1 / 8
    res["masked_elements_per_step"] = elems
    for k, v in t.items():
        us = sum(v) / steps
        gbs = elems * bytes_el / (us * 1e-6) / 1e9
        res[k] = {"launches_per_step": len(v) / steps, "us_per_step": us, "achieved_GBps": gbs, "frac_of_3350_GBps": gbs / 3350.0}
    gan.close(); G.close(); D.close(); ctx.close()
    try:
        res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except Exception as e:
        res["gpu"] = str(e)
    print(json.dumps(res))
    if args.out:
        json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
