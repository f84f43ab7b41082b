"""Cost of the activations of b2g_activation codes 5-16 on bench.py's workloads (bf16, CUDA-graph steps, one GPU).

  C5 and C2 as bench.py runs them (ReLU generator, LeakyReLU(0.2) discriminator), then with every ReLU / LeakyReLU replaced by ELU, then by SELU
  (the output activations stay tanh / XENT):
  1. Step time: `--rounds` alternating runs of `--steps` steps per configuration (CUDA events per step, L2 flushed between steps, as bench.py
     times its configurations), and the kernel launches per step.
  2. The act_ext_* kernels inside each step, timed with torch.profiler (CUDA activities) over 50 replayed steps in a separate run, and their
     algorithmic bytes per step (bf16: 4 B per element forward, z in and a out; 6 B per element backward, z and eps in, eps out) as a fraction of
     the H100 SXM's 3.35 TB/s.
The card's name, power limit and SM clock limit are read in the same process as the timings.
Usage: python tools/activation_bench.py [--steps 100] [--rounds 3] [--out OUT.json]"""
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
from gan_deeplearning4j_b200 import engine, models

KINDS = ("base", "elu", "selu")
HBM_BYTES_PER_S = 3.35e12
LAUNCH_STEPS = 5


def cuda_us(prof, name):
    return [ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            for ev in prof.events() if name in ev.name and ev.device_type == torch.autograd.DeviceType.CUDA]


def specs(cfg, kind):
    if kind == "base":
        return bench.build_specs(cfg)
    if cfg.get("mlp"):
        return (models.mlp_generator(cfg["z"], cfg["hidden"], cfg["d"], activation=kind), models.mlp_discriminator(cfg["d"], cfg["hidden"], activation=kind),
                (cfg["z"],), (cfg["d"],))
    return (models.dcgan_generator(cfg["size"], cfg["z"], cfg["nf"], cfg["nc"], activation=kind),
            models.dcgan_discriminator(cfg["size"], cfg["nf"], cfg["nc"], activation=kind), (cfg["z"],), (cfg["nc"], cfg["size"], cfg["size"]))


def ext_bytes_per_step(net, spec_list, fwd_rows, bwd_rows):
    """Algorithmic bytes of the act_ext kernels of one net per step: its layers of codes 5-16, forwards over fwd_rows rows in all, backwards over
    bwd_rows (bf16: 4 B / element forward, 6 B / element backward)."""
    elems = sum(net.layer_output_size(i) for i, s in enumerate(spec_list) if engine.ACTS[s.get("activation", "identity")] >= 5)
    return elems * (4 * fwd_rows + 6 * bwd_rows)


def make(ctx, cfg_name, kind):
    cfg = bench.CONFIGS[cfg_name]
    gs, ds, gin, din = specs(cfg, kind)
    n = cfg["batch"]
    G = b.Net(ctx, gs, gin, max_batch=n, precision=b.BF16, xent_clip_eps=0.0, seed=666)
    D = b.Net(ctx, ds, din, max_batch=2 * n, precision=b.BF16, xent_clip_eps=0.0, bn_groups=2, seed=667)
    gan = b.Gan(G, D, fake_bn_train=False, use_cuda_graph=True)
    gan.upload(*bench.synthetic(cfg, n, 666))
    # per step: G forward on z_d and on z_g (N rows each), G backward (N); D forward on real|fake (2N) and on G's output (N), D backward on both
    nbytes = ext_bytes_per_step(G, gs, 2 * n, n) + ext_bytes_per_step(D, ds, 3 * n, 3 * n)
    return n, G, D, gan, nbytes


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
    res = {"gpu": gpu, "steps": args.steps, "runs": [], "act_ext_kernels": {}}
    for r in range(args.rounds):
        for cfg_name, kind in cases:
            n, G, D, gan, _ = make(ctx, cfg_name, kind)
            ms = bench.timed_resident_steps(ctx, gan, n, args.steps, 10, ctx.sync)
            l0 = ctx.launch_count()          # launches of graph-replayed steps only, counted around steps of their own
            for _ in range(LAUNCH_STEPS):
                gan.step_resident(n)
            ctx.sync()
            launches = (ctx.launch_count() - l0) / LAUNCH_STEPS
            res["runs"].append({"config": f"{cfg_name}+{kind}", "round": r, "ms_per_step": sum(ms) / len(ms), "samples_per_s": n * len(ms) / (sum(ms) * 1e-3),
                                "launches_per_step": launches, "losses": [float(v) for v in gan.losses()]})
            gan.close(); G.close(); D.close()
    for cfg_name, kind in cases:
        if kind == "base":
            continue
        n, G, D, gan, nbytes = make(ctx, cfg_name, kind)
        for _ in range(10):
            gan.step_resident(n)
        ctx.sync()
        steps = 50
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                gan.step_resident(n)
            ctx.sync()
        fwd, bwd = cuda_us(prof, "act_ext_fwd_kernel"), cuda_us(prof, "act_ext_bwd_kernel")
        us = (sum(fwd) + sum(bwd)) / steps
        res["act_ext_kernels"][f"{cfg_name}+{kind}"] = {"launches_per_step": (len(fwd) + len(bwd)) / steps, "us_per_step": us,
                                                        "fwd_us_per_step": sum(fwd) / steps, "bwd_us_per_step": sum(bwd) / steps,
                                                        "bytes_per_step": nbytes, "fraction_of_3_35_TBps": nbytes / (us * 1e-6) / HBM_BYTES_PER_S if us else None}
        gan.close(); G.close(); D.close()
    ctx.close()
    print(json.dumps(res))
    if args.out:
        json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
