"""PatchGAN discriminators on the H100: C2 / C4 against the same configs with dcgan_discriminator(patch=True), the head conv on its few-output
kernels (impl 5) against the SIMT route (impl 0), and the CnnLossLayer kernels alone.  Prints one JSON object; the card's name, power limit and
max SM clock are part of it.

  python tools/patchgan_bench.py [--steps 50] [--rounds 3] [--out DIR]

Steps: graph-replayed adversarial steps, L2 flushed before each, CUDA-event time per step (b2g_gan_last_step_ms); the configurations alternate
round by round and the table gives the lowest and highest round medians.  Head conv: b2g_test_conv_ex, CUDA events over 20 launches (warm L2).
Loss kernels: torch.profiler (CUDA activity) over 5 calls through b2g_test_ew, algorithmic bytes = z + dz (2 B each in bf16) + labels (4 B)
per element, share of the data sheet's 3.35 TB/s."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import gan_deeplearning4j_b200 as b                      # noqa: E402
from gan_deeplearning4j_b200 import models as m           # noqa: E402

CONFIGS = {"c2": dict(size=64, z=100, nf=64, batch=128), "c4": dict(size=128, z=100, nf=64, batch=32)}
HBM = 3.35e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                              check=True).stdout.strip()
    except Exception as e:          # the numbers are still taken; the card line says why it is missing
        return f"unavailable: {e}"


def make_gan(ctx, cfg, patch):
    size, z, nf, n = cfg["size"], cfg["z"], cfg["nf"], cfg["batch"]
    G = b.Net(ctx, m.dcgan_generator(size, z, nf, 3), (z,), max_batch=n, precision=b.BF16)
    D = b.Net(ctx, m.dcgan_discriminator(size, nf, 3, patch=patch), (3, size, size), max_batch=2 * n, precision=b.BF16, bn_groups=2)
    gan = b.Gan(G, D, use_cuda_graph=True)
    rng = np.random.default_rng(0)
    x = rng.uniform(-1, 1, (n, 3, size, size)).astype(np.float32)
    zd, zg = rng.uniform(-1, 1, (n, z)).astype(np.float32), rng.uniform(-1, 1, (n, z)).astype(np.float32)
    gan.upload(x, zd, zg, np.ones(n, np.float32), np.zeros(n, np.float32), np.ones(n, np.float32))
    return G, D, gan


def time_steps(ctx, G, D, gan, n, steps):
    ms = []
    for _ in range(steps):
        ctx.flush_l2()
        gan.step_resident(n)
        ms.append(gan.last_step_ms())
    return float(np.median(ms))


def counts(ctx, G, D, gan, n, steps=5):
    ctx.sync(); l0, s0 = ctx.launch_count(), G.simt_gemm_calls() + D.simt_gemm_calls()
    for _ in range(steps):
        gan.step_resident(n)
    ctx.sync()
    return (ctx.launch_count() - l0) / steps, (G.simt_gemm_calls() + D.simt_gemm_calls() - s0) / steps


def head_geom(cfg, patch_n):
    side = max(4, cfg["size"] // 16)
    c = cfg["nf"] * 2 ** (min(int(np.log2(cfg["size"])) - 2, 4) - 1)
    return dict(n=patch_n, h=side, w=side, c=c, oh=side, ow=side, o=1, kh=3, kw=3, sh=1, sw=1, ph=1, pw=1)


def head_times(ctx, g):
    rng = np.random.default_rng(1)
    nx, ny, nw = g["n"] * g["h"] * g["w"] * g["c"], g["n"] * g["oh"] * g["ow"] * g["o"], g["o"] * 9 * g["c"]
    x, dy, w = rng.uniform(-1, 1, nx), rng.uniform(-1, 1, ny), rng.uniform(-1, 1, nw)
    out = {}
    for impl in (0, 5):
        for kind, a, bb, size in ((0, x, w, ny), (1, dy, w, nx), (2, x, dy, nw)):
            _, _, kern, ms = b.test_conv_ex(ctx, kind, g, a, bb, size, impl=impl, iters=20)
            out[f"impl{impl}_{['fprop', 'dgrad', 'wgrad'][kind]}"] = {"kernel": kern, "us": round(ms * 1e3, 2)}
    return out


def loss_kernel_times(ctx, out_dir):
    from torch.profiler import ProfilerActivity, profile
    cases = {"cnn_xent C2 patch D step (2 x 128 x 16)": ("cnn_xent", 2, 128 * 16, 1),
             "cnn_xent 2 x 64 x 64 x 64 map": ("cnn_xent", 2, 64 * 64 * 64, 1),
             "cnn_softmax_xent 16 x 128 x 128 pixels, C = 21": ("cnn_softmax_xent", 1, 16 * 128 * 128, 21)}
    res = {}
    for name, (op, groups, rows, c) in cases.items():
        n = groups * rows * c
        rng = np.random.default_rng(2)
        z, y = rng.uniform(-3, 3, n).astype(np.float32), rng.uniform(0, 1, n).astype(np.float32)
        b.test_ew(ctx, b.BF16, op, z, y, (0, 0, 0), rows=rows, cols=c, groups=groups)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                b.test_ew(ctx, b.BF16, op, z, y, (0, 0, 0), rows=rows, cols=c, groups=groups)
        evs = [e for e in prof.key_averages() if f"{op}_kernel" in e.key]
        us = sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) for e in evs) / max(1, sum(e.count for e in evs))
        byts = n * (2 + 2 + 4)
        res[name] = {"us": round(us, 2), "algorithmic_bytes": byts, "share_of_3.35TB/s": round(byts / (us * 1e-6) / HBM, 4) if us else None}
        if out_dir:
            prof.export_chrome_trace(os.path.join(out_dir, f"patchgan_{op}_{rows}.json"))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    ap.add_argument("--loss-only", action="store_true", help="only the loss kernels")
    a = ap.parse_args()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
    ctx = b.Context(0)
    res = {"card": card(), "steps": {}, "head_conv": {}, "loss_kernels": {}}
    for name, cfg in ({} if a.loss_only else CONFIGS).items():
        nets = {p: make_gan(ctx, cfg, p) for p in (False, True)}
        rounds = {p: [] for p in nets}
        for p, (G, D, gan) in nets.items():
            time_steps(ctx, G, D, gan, cfg["batch"], 5)          # capture and warm up
        for _ in range(a.rounds):
            for p, (G, D, gan) in nets.items():
                rounds[p].append(time_steps(ctx, G, D, gan, cfg["batch"], a.steps))
        for p, (G, D, gan) in nets.items():
            launches, simt = counts(ctx, G, D, gan, cfg["batch"])
            key = name + ("_patch" if p else "")
            res["steps"][key] = {"ms_per_step": [round(min(rounds[p]), 4), round(max(rounds[p]), 4)], "launches_per_step": launches, "simt_calls_per_step": simt}
            gan.close(); G.close(); D.close()
        res["head_conv"][name + "_patch (D step, 2N)"] = {"geom": head_geom(cfg, 2 * cfg["batch"]), **head_times(ctx, head_geom(cfg, 2 * cfg["batch"]))}
    res["loss_kernels"] = loss_kernel_times(ctx, a.out)
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
