"""Cost of DL4J's weight constraints on bench.py's workloads (bf16, CUDA-graph steps, one GPU).

  C2 and C5 against the same configurations with MaxNorm per output unit on every W of G and D (conv W dims {1, 2, 3}, deconv W {0, 2, 3},
  dense / output W {0}; bound 1.0):
  1. Step time, `--rounds` alternating runs of `--steps` steps per configuration (CUDA events per step, L2 flushed between steps, as bench.py
     times its configurations), and the kernel launches per step.
  2. The constraint kernels inside each constrained step, timed with torch.profiler (CUDA activities) over 50 replayed steps in a separate
     run, and their algorithmic bytes over kernel time against the H100 SXM data-sheet 3.35 TB/s.  Bytes per constrained parameter: 10 on the
     one-pass path (read 4, write 4, bf16 copy 2), 14 on the two-launch path (norm read 4, scale read 4 + write 4, bf16 copy 2); the packed
     pixel-shuffle copy (2 B for G's last W only) and the per-group partials are left out.
  3. Which tensors take which path (the rule stated at b2g_constraint in include/b200gan.h).
The card's name, power limit and SM clock limit are read in the same process as the timings.
Usage: python tools/constraint_bench.py [--steps 100] [--rounds 3] [--out OUT.json]"""
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

CASES = (("c5", False), ("c5", True), ("c2", False), ("c2", True))
PER_UNIT = {"conv2d": (1, 2, 3), "deconv2d": (0, 2, 3), "dense": (0,), "output": (0,)}
BOUND = 1.0


def with_n_in(net):
    """The net's GEMM specs with n_in filled in where it is inferred (the MLP's dense layers take the previous one's features)."""
    out, cur = [], 1
    for d in net.input_shape:
        cur *= d
    for sp in net.specs:
        if sp["type"] in PER_UNIT:
            sp = dict(sp, n_in=sp.get("n_in") or cur)
            out.append(sp)
            cur = sp["n_out"]
    return out


def path(spec):
    """(path, parameters) of a W under MaxNorm per output unit: one-pass when the innermost stored axis (nIn of a conv / dense W) is reduced
    and a group holds <= 4096 elements; a deconv W per output unit keeps its innermost nOut axis (strided groups) and takes two launches."""
    k = spec.get("kernel", (1, 1)) if spec["type"] in ("conv2d", "deconv2d") else (1, 1)
    n = spec["n_in"] * spec["n_out"] * k[0] * k[1]
    one = spec["type"] != "deconv2d" and spec["n_in"] * k[0] * k[1] <= 4096
    return ("one-pass" if one else "two-launch"), n


def constrain(net):
    for sp in net.specs:
        if sp["type"] in PER_UNIT:
            net.set_constraints([m.max_norm(BOUND, PER_UNIT[sp["type"]])], sp["name"])


def make(ctx, cfg_name, on):
    cfg = bench.CONFIGS[cfg_name]
    G, D, gan = bench.make_gan(b, ctx, cfg, cfg["batch"])
    if on:
        constrain(G); constrain(D)
    gan.upload(*bench.synthetic(cfg, cfg["batch"], 666))
    return cfg["batch"], G, D, gan


def name(cfg_name, on):
    return cfg_name + ("+maxnorm" if on else "")


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
    res = {"gpu": gpu, "steps": args.steps, "runs": [], "constraint_kernels": {}, "paths": {}}
    for r in range(args.rounds):
        for cfg_name, on in CASES:
            n, G, D, gan = make(ctx, cfg_name, on)
            l0 = ctx.launch_count()
            ms = bench.timed_resident_steps(ctx, gan, n, args.steps, 10, ctx.sync)
            launches = (ctx.launch_count() - l0) / (args.steps + max(3, 10))
            res["runs"].append({"config": name(cfg_name, on), "round": r, "ms_per_step": sum(ms) / len(ms), "samples_per_s": n * len(ms) / (sum(ms) * 1e-3),
                                "launches_per_step": launches})
            gan.close(); G.close(); D.close()
    for cfg_name, on in CASES:
        if not on:
            continue
        n, G, D, gan = make(ctx, cfg_name, on)
        tensors = {sp["name"]: path(sp) for net in (G, D) for sp in with_n_in(net)}
        res["paths"][cfg_name] = {k: {"path": p, "params": c} for k, (p, c) in tensors.items()}
        byts = sum((10 if p == "one-pass" else 14) * c for p, c in tensors.values())
        for _ in range(10):
            gan.step_resident(n)
        ctx.sync()
        steps = 50
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                gan.step_resident(n)
            ctx.sync()
        evs = [ev for ev in prof.events() if "constraint_" in ev.name and ev.device_type == torch.autograd.DeviceType.CUDA]
        t = lambda ev: ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        per_kernel = {}
        for ev in evs:
            k = ev.name.split("(")[0].split("::")[-1]
            per_kernel[k] = per_kernel.get(k, 0.0) + t(ev) / steps
        us = sum(per_kernel.values())
        gbs = byts / (us * 1e-6) / 1e9 if us > 0 else 0.0
        res["constraint_kernels"][name(cfg_name, on)] = {"launches_per_step": len(evs) / steps, "us_per_step": us, "us_per_kernel": per_kernel,
                                                         "constrained_params": sum(c for _, c in tensors.values()), "algorithmic_MB_per_step": byts / 1e6,
                                                         "achieved_GBps": gbs, "frac_of_3350_GBps": gbs / 3350.0}
        gan.close(); G.close(); D.close()
    ctx.close()
    print(json.dumps(res))
    if args.out:
        json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
