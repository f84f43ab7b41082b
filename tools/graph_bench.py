"""Skip connections on the H100: the residual C2 adversarial step beside the plain C2 step, a U-Net training step, and the vertex kernels alone.
Prints one JSON object; the card's name, power limit and max SM clock are part of it.

  python tools/graph_bench.py [--steps 50] [--rounds 3] [--out DIR]

Steps: graph-replayed adversarial steps (C2: 64x64x3, z = 100, nf = 64, batch 128, bf16), L2 flushed before each, CUDA-event time per step
(b2g_gan_last_step_ms); the plain and residual (dcgan_*(residual=True)) configurations alternate round by round and the table gives the lowest
and highest round medians, with launches and SIMT GEMM calls per step.  U-Net: models.unet(64, 3, 2 classes, nf = 32, depth 2) bf16 fit at
batch 128, host clock around a synchronised fit, SIMT GEMM calls per fit.  Vertex kernels: torch.profiler (CUDA activity) over 5 calls through
b2g_test_ew at the sizes the two workloads run them, algorithmic bytes per call over kernel time as a share of the data sheet's 3.35 TB/s."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import gan_deeplearning4j_b200 as b                      # noqa: E402
from gan_deeplearning4j_b200 import models as m           # noqa: E402

C2 = dict(size=64, z=100, nf=64, batch=128)
HBM = 3.35e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                              check=True).stdout.strip()
    except Exception as e:          # the numbers are still taken; the card line says why it is missing
        return f"unavailable: {e}"


def make_gan(ctx, residual):
    size, z, nf, n = C2["size"], C2["z"], C2["nf"], C2["batch"]
    G = b.Net(ctx, m.dcgan_generator(size, z, nf, 3, residual=residual), (z,), max_batch=n, precision=b.BF16)
    D = b.Net(ctx, m.dcgan_discriminator(size, nf, 3, residual=residual), (3, size, size), max_batch=2 * n, precision=b.BF16, bn_groups=2)
    gan = b.Gan(G, D, use_cuda_graph=True)
    rng = np.random.default_rng(0)
    x = rng.uniform(-1, 1, (n, 3, size, size)).astype(np.float32)
    zd, zg = rng.uniform(-1, 1, (n, z)).astype(np.float32), rng.uniform(-1, 1, (n, z)).astype(np.float32)
    gan.upload(x, zd, zg, np.ones(n, np.float32), np.zeros(n, np.float32), np.ones(n, np.float32))
    return G, D, gan


def time_steps(ctx, gan, n, steps):
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


def unet_step(ctx, steps):
    n, size = 128, 64
    net = b.Net(ctx, m.unet(size, 3, 2, 32, 2), (3, size, size), max_batch=n, precision=b.BF16)
    rng = np.random.default_rng(1)
    x = rng.uniform(-1, 1, (n, 3, size, size)).astype(np.float32)
    lab = rng.integers(0, 2, (n, size, size))
    y = np.ascontiguousarray(np.moveaxis(np.eye(2, dtype=np.float32)[lab], -1, 1))
    for _ in range(3):
        net.fit(x, y)
    s0, l0 = net.simt_gemm_calls(), ctx.launch_count()
    t0 = time.perf_counter()
    for _ in range(steps):
        net.fit(x, y)                    # returns after a device synchronise
    ms = (time.perf_counter() - t0) * 1e3 / steps
    res = {"ms_per_fit_incl_host_copies": round(ms, 3), "simt_calls_per_fit": (net.simt_gemm_calls() - s0) / steps,
           "launches_per_fit": (ctx.launch_count() - l0) / steps}
    net.close()
    return res


def vertex_kernel_times(ctx, out_dir):
    from torch.profiler import ProfilerActivity, profile
    # (label, op, test_ew arguments, kernel name, algorithmic bytes per call in bf16)
    n_g = 128 * 32 * 32 * 64                  # the generator's last residual block (32x32x64, N = 128)
    n_d = 256 * 32 * 32 * 64                  # the discriminator's first residual block in the D step (32x32x64, 2N = 256)
    px, c = 128 * 64 * 64, 32                 # the U-Net's top merge (64x64, 32 + 32 channels, N = 128)
    cases = [("Add forward, D block 1 (2N)", "vertex_fwd", dict(n=n_d), n_d, n_d, "vertex_ew_fwd_kernel", 3 * 2 * n_d),
             ("Add backward, D block 1 (2N)", "vertex_bwd", dict(n=n_d), 2 * n_d, 2 * n_d, "vertex_ew_bwd_kernel", n_d * (2 + 4)),
             ("skip add, D block 1 source (2N)", "skip_add", dict(n=n_d), n_d, n_d, "skip_add_kernel", n_d * (2 + 4 + 2)),
             ("Add forward, G block 4 (N)", "vertex_fwd", dict(n=n_g), n_g, n_g, "vertex_ew_fwd_kernel", 3 * 2 * n_g),
             ("Merge forward, U-Net top (N)", "merge_fwd", dict(rows=px, cols=c, C=c), px * c, px * c, "merge_fwd_kernel", 2 * 2 * px * 2 * c),
             ("Merge backward, U-Net top (N)", "merge_bwd", dict(rows=px, cols=c, C=c), px * 2 * c, 0, "merge_bwd_kernel", px * 2 * c * 2 + px * c * (2 + 4))]
    res = {}
    rng = np.random.default_rng(2)
    for label, op, kw, n0, n1, kname, byts in cases:
        a = rng.uniform(-1, 1, n0).astype(np.float32)
        bb = rng.uniform(-1, 1, n1).astype(np.float32) if n1 else None
        extra = {"act": "add"} if op.startswith("vertex") else {}
        b.test_ew(ctx, b.BF16, op, a, bb, (0, 0, 0), **extra, **kw)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                b.test_ew(ctx, b.BF16, op, a, bb, (0, 0, 0), **extra, **kw)
        evs = [e for e in prof.key_averages() if kname in e.key]
        us = sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) for e in evs) / max(1, sum(e.count for e in evs))
        res[label] = {"kernel": kname, "us": round(us, 2), "algorithmic_bytes": byts, "share_of_3.35TB/s": round(byts / (us * 1e-6) / HBM, 4) if us else None}
        if out_dir:
            prof.export_chrome_trace(os.path.join(out_dir, f"graph_{op}_{n0}.json"))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
    ctx = b.Context(0)
    res = {"card": card(), "steps": {}, "unet": {}, "vertex_kernels": {}}
    nets = {r: make_gan(ctx, r) for r in (False, True)}
    rounds = {r: [] for r in nets}
    for r, (G, D, gan) in nets.items():
        time_steps(ctx, gan, C2["batch"], 5)                  # capture and warm up
    for _ in range(a.rounds):
        for r, (G, D, gan) in nets.items():
            rounds[r].append(time_steps(ctx, gan, C2["batch"], a.steps))
    for r, (G, D, gan) in nets.items():
        launches, simt = counts(ctx, G, D, gan, C2["batch"])
        res["steps"]["c2_residual" if r else "c2"] = {"ms_per_step": [round(min(rounds[r]), 4), round(max(rounds[r]), 4)], "launches_per_step": launches,
                                                      "simt_calls_per_step": simt}
        gan.close(); G.close(); D.close()
    res["unet"] = unet_step(ctx, max(5, a.steps // 5))
    res["vertex_kernels"] = vertex_kernel_times(ctx, a.out)
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
