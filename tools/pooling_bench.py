"""Cost of average, sum and p-norm pooling (bf16, one GPU).

  1. C2 as bench.py runs it against C2 with a global-pooling-head discriminator (GlobalPoolingLayer SUM / AVG + OutputLayer(nOut 1) in place of
     the last 4x4 valid conv and its LossLayer): `--rounds` alternating runs of `--steps` graph-replayed steps per configuration (CUDA events per
     step, L2 flushed between steps, as bench.py times its configurations), and the kernel launches per step.
  2. Each new kernel with torch.profiler (CUDA activities) in a separate run, through its production wrapper (b2g_test_pool ops pool2d /
     global_pool, `--reps` calls per case, median device time): SubsamplingLayer AVG / PNORM(2) 2x2 s2 on [256, 32, 32, 64] and [256, 16, 16, 128],
     GlobalPoolingLayer MAX / AVG / PNORM(2) on [256, 4, 4, 512] and [32, 64, 64, 128], all NHWC bf16.  The hook writes the inputs on the device
     right before the forward, so part of them may still sit in L2.  Algorithmic bytes come from the shapes (below) and are reported over
     the kernel time as a fraction of the H100 SXM's 3.35 TB/s.
The card's name, power limit and SM clock limit are read in the same process as the timings.
Usage: python tools/pooling_bench.py [--steps 100] [--rounds 3] [--reps 5] [--out OUT.json]"""
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

HEADS = ("base", "sum", "avg")
HBM_BYTES_PER_S = 3.35e12
LAUNCH_STEPS = 5
TS = 2                          # bf16 bytes
SUB_SHAPES = [(256, 32, 32, 64), (256, 16, 16, 128)]
GLOBAL_SHAPES = [(256, 4, 4, 512), (32, 64, 64, 128)]


def cuda_us(prof, name):
    return [ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            for ev in prof.events() if name in ev.name and ev.device_type == torch.autograd.DeviceType.CUDA]


def pool2d_bytes(kind, n, h, w, c):
    """2x2 s2: forward reads x, writes y; backward reads eps_out, writes eps_in, and PNORM also reads x and y."""
    xi, yo = n * h * w * c * TS, n * (h // 2) * (w // 2) * c * TS
    return xi + yo, yo + xi + (xi + yo if kind == "pnorm" else 0)


def global_bytes(kind, n, h, w, c):
    """forward reads x, writes y (MAX also its int32 index); backward reads eps_out (and MAX's index, PNORM's y and x), writes eps_in."""
    xi, yo = n * h * w * c * TS, n * c * TS
    fwd = xi + yo + (n * c * 4 if kind == "max" else 0)
    bwd = yo + xi + {"max": n * c * 4, "pnorm": yo + xi}.get(kind, 0)
    return fwd, bwd


def make(ctx, head):
    cfg = bench.CONFIGS["c2"]
    gs, ds, gin, din = bench.build_specs(cfg)
    if head != "base":
        ds = models.dcgan_discriminator(cfg["size"], cfg["nf"], cfg["nc"], global_pooling=head)
    n = cfg["batch"]
    G = b.Net(ctx, gs, gin, max_batch=n, precision=b.BF16, xent_clip_eps=0.0, seed=666)
    D = b.Net(ctx, ds, din, max_batch=2 * n, precision=b.BF16, xent_clip_eps=0.0, bn_groups=2, seed=667)
    gan = b.Gan(G, D, fake_bn_train=False, use_cuda_graph=True)
    gan.upload(*bench.synthetic(cfg, n, 666))
    return n, G, D, gan


def kernel_case(ctx, op, kind, shape, reps):
    n, h, w, c = shape
    rng = np.random.default_rng(0)
    x = rng.uniform(-1, 1, shape).astype(np.float32)
    if op == "pool2d":
        e = rng.uniform(-1, 1, (n, h // 2, w // 2, c)).astype(np.float32)
        kw = dict(KH=2, KW=2, SH=2, SW=2)
        fb, bb = pool2d_bytes(kind, *shape)
    else:
        e = rng.uniform(-1, 1, (n, c)).astype(np.float32)
        kw = {}
        fb, bb = global_bytes(kind, *shape)
    call = lambda: b.test_pool(ctx, b.BF16, op, x, e, (0, 0, 0), pooling=kind, N=n, H=h, W=w, C=c, pnorm=2.0, **kw)
    _, info = call()                                                          # warm-up (and the split count)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            ctx.flush_l2()
            call()
        ctx.sync()
    fwd, bwd = cuda_us(prof, f"{op}_fwd_kernel"), cuda_us(prof, f"{op}_bwd_kernel")
    out = {"op": op, "kind": kind, "shape_nhwc": list(shape), "kernels": info["kernel"], "global_splits": info["splits"] if op == "global_pool" else None}
    for name, times, nbytes in (("fwd", fwd, fb), ("bwd", bwd, bb)):
        us = float(np.median(times)) if times else None
        out[name] = {"us": us, "calls": len(times), "bytes": nbytes, "GBps": nbytes / (us * 1e-6) / 1e9 if us else None,
                     "fraction_of_3_35_TBps": nbytes / (us * 1e-6) / HBM_BYTES_PER_S if us else None}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except Exception as e:
        gpu = str(e)
    ctx = b.Context(0)
    res = {"gpu": gpu, "steps": args.steps, "runs": [], "kernels": []}
    for r in range(args.rounds):
        for head in HEADS:
            n, G, D, gan = make(ctx, head)
            ms = bench.timed_resident_steps(ctx, gan, n, args.steps, 10, ctx.sync)
            l0 = ctx.launch_count()          # launches of graph-replayed steps only, counted around steps of their own
            for _ in range(LAUNCH_STEPS):
                gan.step_resident(n)
            ctx.sync()
            launches = (ctx.launch_count() - l0) / LAUNCH_STEPS
            res["runs"].append({"config": f"c2+{head}", "round": r, "ms_per_step": sum(ms) / len(ms), "samples_per_s": n * len(ms) / (sum(ms) * 1e-3),
                                "launches_per_step": launches, "losses": [float(v) for v in gan.losses()]})
            gan.close(); G.close(); D.close()
    for shape in SUB_SHAPES:
        for kind in ("avg", "pnorm"):
            res["kernels"].append(kernel_case(ctx, "pool2d", kind, shape, args.reps))
    for shape in GLOBAL_SHAPES:
        for kind in ("max", "avg", "pnorm"):
            res["kernels"].append(kernel_case(ctx, "global_pool", kind, shape, args.reps))
    ctx.close()
    print(json.dumps(res))
    if args.out:
        json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
