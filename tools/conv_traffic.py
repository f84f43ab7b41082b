"""Where the tensor-core GEMM time of a DCGAN step goes, set against the operand bytes each launch pulls from L2.

  1. Every row of bench.gemm_family (the step's tensor-core GEMM launches) timed alone through the kernel-level hook, as bench.py times its
     `roofline_family` (CUDA events, warm L2, --iters launches), with the kernel label, whether the launch ran the slab path, and the A and B
     operand bytes its TMA boxes load, from the byte model below.  bytes / time is the operand delivery rate of the launch.
     --per-tap times the 4x4 s2 p1 fprop / dgrad launches on one activation box per tap (the path the slabs replaced), for a before / after
     comparison in one session.
  2. torch.profiler (CUDA activities) over --steps graph-replayed steps of the same configuration: every kernel of the step with its launches
     and microseconds per step; the trace goes under --out.
The card name, power limit and maximum SM clock are read in the same run.

Byte model (mirror of kernels_tc.cu's host-side tiling, kept here with the tool):
  tc_conv_kernel per tap    work items x taps x chunks K-blocks, each one 128-row x 64-channel activation box (16 KB) + a BN x 64 weight tile
  tc_conv_kernel slab       work items x (row pairs x column taps x chunks) K units, each one slab box of Nt x (Ht+1) x Wt rows x 128 B + two
                            weight tiles; row pairs = 2 (fprop) / 1 (dgrad phase), column taps = 4 / 2
  tc_wgrad_kernel           per (128 output channels x BNW columns) CTA column, every 64-pixel K-block once: a 2 x 64 x 64 dy box (16 KB) +
                            BNW / 64 activation boxes of 64 x 64
Usage: python tools/conv_traffic.py [--config c2] [--iters 20] [--steps 20] [--per-tap] [--out DIR]"""
import argparse
import collections
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np

import bench
import gan_deeplearning4j_b200 as b

SLAB_ROWS = 144      # kernels_tc.cu SLAB_ROWS


def row_tile(n, gh, gw, rows=128):
    p = gh * gw
    if gw > rows or rows % gw:
        return None
    if p >= rows:
        ht = rows // gw
        return (1, ht, gw) if p % rows == 0 and gh % ht == 0 else None
    if rows % p or n % (rows // p):
        return None
    return rows // p, gh, gw


def pick_bn_fill(oc, m_tiles_x_phases, sms):
    bn = 128 if oc % 128 == 0 else 64
    while bn > 64 and m_tiles_x_phases * (oc // bn) < sms:
        bn //= 2
    return bn


def slab_applies(nt, ht, wt, bn):
    return bn == 64 and wt % 8 == 0 and ((nt == 1 and ht >= 2) or (nt == 2 and ht * wt == 64)) and nt * (ht + 1) * wt <= SLAB_ROWS


def conv_bytes(kind, n, h, c, o, sms, slab):
    """(A bytes, B bytes) of one tc_conv_kernel launch of the 4x4 s2 p1 geometry x [n,h,h,c] -> y [n,h/2,h/2,o]; kind 0 fprop, 1 dgrad;
    slab: the launch ran the slab path (slab_applies says where the kernel takes it)."""
    g = h // 2
    nt, ht, wt = row_tile(n, g, g)
    tiles_m = n * g * g // 128
    if kind == 0:
        phases, oc, chunks, taps, pairs, cols = 1, o, c // 64, 16, 2, 4
    else:
        phases, oc, chunks, taps, pairs, cols = 4, c, o // 64, 4, 1, 2
    bn = pick_bn_fill(oc, tiles_m * phases, sms)
    items = tiles_m * (oc // bn) * phases
    if slab:
        assert slab_applies(nt, ht, wt, bn), "the byte model does not know this slab shape"
        units = pairs * cols * chunks
        return items * units * nt * (ht + 1) * wt * 128, items * units * 2 * bn * 128
    kbs = taps * chunks
    return items * kbs * 128 * 128, items * kbs * bn * 128


def wgrad_bytes(n, h, c, o):
    g = h // 2
    bnw = 128 if (16 * c) % 128 == 0 else 64
    cols, otiles, kb_total = 16 * c // bnw, o // 128, n * g * g // 64
    return kb_total * 16384 * cols * otiles, kb_total * bnw * 128 * cols * otiles


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip()
    except Exception as e:     # pragma: no cover
        return str(e)


def launch_table(ctx, cfg, iters, per_tap, sms):
    rng = np.random.default_rng(0)
    rows, cache = [], {}
    for name, kind, n, h, c, o, count in bench.gemm_family(cfg, cfg["batch"]):
        geom = dict(n=n, h=h, w=h, c=c, oh=h // 2, ow=h // 2, o=o, kh=4, kw=4, sh=2, sw=2, ph=1, pw=1)
        nx, ny, nw = n * h * h * c, n * (h // 2) * (h // 2) * o, o * 16 * c
        key = (kind, n, h, c, o)
        if key not in cache:
            a = rng.standard_normal(ny if kind == 1 else nx, dtype=np.float32)
            bb = rng.standard_normal(ny if kind == 2 else nw, dtype=np.float32) * 0.05
            if kind == 2:
                _, ms = b.test_conv(ctx, 2, 1, b.BF16, geom, a, bb, nw, iters=iters)
                kern, (ab, bbytes), slab = "tc_wgrad", wgrad_bytes(n, h, c, o), False
            else:
                info = {}
                try:
                    _, _, kern, ms = b.test_conv_ex(ctx, kind, geom, a, bb, ny if kind == 0 else nx, iters=iters, per_tap=per_tap, info=info)
                except TypeError:        # a library from before the slab path (before / after comparisons): every launch is per tap
                    assert not per_tap
                    _, _, kern, ms = b.test_conv_ex(ctx, kind, geom, a, bb, ny if kind == 0 else nx, iters=iters)
                slab = info.get("slab", False)
                ab, bbytes = conv_bytes(kind, n, h, c, o, sms, slab)
            cache[key] = (ms, kern, ab, bbytes, slab)
        ms, kern, ab, bbytes, slab = cache[key]
        rows.append(dict(name=name, kernel=kern, slab=slab, count=count, us=ms * 1e3, a_mb=ab / 1e6, b_mb=bbytes / 1e6,
                         gbs=(ab + bbytes) / (ms * 1e-3) / 1e9))
    return rows


def profile_step(ctx, cfg, steps, out_dir):
    import torch
    n = cfg["batch"]
    G, D, gan = bench.make_gan(b, ctx, cfg, n)
    gan.upload(*bench.synthetic(cfg, n, 666))
    for _ in range(10):
        gan.step_resident(n)
    ctx.sync()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            gan.step_resident(n)
        ctx.sync()
    prof.export_chrome_trace(os.path.join(out_dir, "step.pt.trace.json"))
    agg = collections.defaultdict(lambda: [0, 0.0])
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            agg[ev.name][0] += 1
            agg[ev.name][1] += t
    gan.close(); G.close(); D.close()
    return sorted(({"kernel": k, "launches_per_step": v[0] / steps, "us_per_step": v[1] / steps} for k, v in agg.items()),
                  key=lambda r: -r["us_per_step"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="c2", choices=[k for k, v in bench.CONFIGS.items() if not v.get("mlp")])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--per-tap", dest="per_tap", action="store_true")
    ap.add_argument("--out", default="conv_traffic_out")
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cfg = bench.CONFIGS[args.config]
    ctx = b.Context(0)
    res = {"gpu": gpu_info(), "config": args.config, "per_tap": args.per_tap, "iters": args.iters}
    rows = launch_table(ctx, cfg, args.iters, args.per_tap, sms)
    res["launches"] = rows
    res["ms_per_step_if_serialised"] = sum(r["us"] * r["count"] for r in rows) / 1e3
    res["operand_gb_per_step"] = sum((r["a_mb"] + r["b_mb"]) * r["count"] for r in rows) / 1e3
    print(f"# {res['gpu']}  config {args.config}{'  (per-tap activation loads)' if args.per_tap else ''}")
    print(f"{'launch':58s} {'kernel':24s} slab {'us':>7s} {'A MB':>7s} {'B MB':>7s} {'GB/s':>7s}")
    for r in rows:
        print(f"{r['name'][:58]:58s} {r['kernel'][:24]:24s} {'yes ' if r['slab'] else 'no  '} {r['us']:7.1f} {r['a_mb']:7.1f} {r['b_mb']:7.1f} {r['gbs']:7.0f}")
    print(f"serialised: {res['ms_per_step_if_serialised']:.4f} ms per step, operands {res['operand_gb_per_step']:.3f} GB per step")
    if args.steps > 0:
        res["step_kernels"] = profile_step(ctx, cfg, args.steps, args.out)
        print(f"\n# kernels of the {args.config} step (torch.profiler, {args.steps} graph-replayed steps, L2 not flushed)")
        for r in res["step_kernels"]:
            print(f"{r['us_per_step']:9.1f} us {r['launches_per_step']:5.1f} x  {r['kernel'][:110]}")
        print(f"total {sum(r['us_per_step'] for r in res['step_kernels']):.1f} us of kernel time per step")
    ctx.close()
    with open(os.path.join(args.out, f"conv_traffic_{args.config}{'_per_tap' if args.per_tap else ''}.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
