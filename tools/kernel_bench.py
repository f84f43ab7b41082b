"""Time every tensor-core GEMM shape of the C2 step in isolation (CUDA events inside b2g_test_conv, 20 iterations, warm L2)
and print achieved TFLOP/s against MEASURED_PEAKS.json.  usage: python tools/kernel_bench.py [batch]"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np

import gan_deeplearning4j_b200 as b

edge_only = "--edge-only" in sys.argv
args = [a for a in sys.argv[1:] if not a.startswith("--")]
n = int(args[0]) if args else 128
peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["bf16_tflops"] if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else 989.0      # H100 SXM data-sheet dense bf16
ctx = b.Context(0)
rng = np.random.default_rng(0)
# (name, kind, batch, h, w, c, o)  conv geometry 4x4 s2 p1; kind 0 fprop, 1 dgrad(=deconv fwd), 2 wgrad
shapes = []
for name, bt, h, c, o in (("D2", 2 * n, 32, 64, 128), ("D3", 2 * n, 16, 128, 256), ("D4", 2 * n, 8, 256, 512)):
    shapes += [(name + " fprop (D-step 2N)", 0, bt, h, h, c, o), (name + " wgrad (D-step 2N)", 2, bt, h, h, c, o), (name + " dgrad (G-step N)", 1, n, h, h, c, o)]
for name, h, c, o in (("G2", 8, 256, 512), ("G3", 16, 128, 256), ("G4", 32, 64, 128)):   # conv-equivalent geometry of the transposed convs
    shapes += [(name + " fwd = dgrad form (N)", 1, n, h, h, c, o), (name + " wgrad (N)", 2, n, h, h, c, o), (name + " input-grad = fprop form (N)", 0, n, h, h, c, o)]
# skinny layers (3 image channels): impl 2 = SIMT, impl 3 = tensor cores; (name, kind, batch)
edge = [("D1 fprop (D-step 2N)", 0, 2 * n), ("D1 wgrad (D-step 2N)", 2, 2 * n), ("D1 dgrad (G-step N)", 1, n),
        ("G5 fwd = dgrad form (N)", 1, n), ("G5 wgrad (N)", 2, n), ("G5 input-grad = fprop form (N)", 0, n)]
edge_rows = []
for name, kind, bt in edge:
    h = w = 64; c = 3; o = 64
    g = dict(n=bt, h=h, w=w, c=c, oh=h // 2, ow=w // 2, o=o, kh=4, kw=4, sh=2, sw=2, ph=1, pw=1)
    nx, ny, nw = bt * h * w * c, bt * (h // 2) * (w // 2) * o, o * 16 * c
    a = rng.standard_normal(ny if kind == 1 else nx, dtype=np.float32)
    bb = rng.standard_normal(ny if kind == 2 else nw, dtype=np.float32) * 0.05
    out_size = ny if kind == 0 else nx if kind == 1 else nw
    t = []
    for impl in (2, 3):
        try:
            _, ms = b.test_conv(ctx, kind, impl, b.BF16, g, a, bb, out_size, iters=20); t.append(ms * 1e3)
        except b.B200GanError:
            t.append(float("nan"))
    edge_rows.append((name, 2.0 * bt * (h // 2) * (w // 2) * o * 16 * c / 1e9, (nx + ny) * 2 / 1e6, t[0], t[1]))
rows = []
for name, kind, bt, h, w, c, o in ([] if edge_only else shapes):
    g = dict(n=bt, h=h, w=w, c=c, oh=h // 2, ow=w // 2, o=o, kh=4, kw=4, sh=2, sw=2, ph=1, pw=1)
    nx, ny, nw = bt * h * w * c, bt * (h // 2) * (w // 2) * o, o * 16 * c
    a = rng.standard_normal(ny if kind == 1 else nx, dtype=np.float32)
    bb = rng.standard_normal(ny if kind == 2 else nw, dtype=np.float32) * 0.05
    out_size = ny if kind == 0 else nx if kind == 1 else nw
    flops = 2.0 * bt * (h // 2) * (w // 2) * o * 16 * c
    try:
        _, ms = b.test_conv(ctx, kind, 1, b.BF16, g, a, bb, out_size, iters=20)
        rows.append((name, flops / 1e9, ms * 1e3, flops / ms / 1e9, flops / ms / 1e9 / peak))
    except b.B200GanError as e:
        rows.append((name, flops / 1e9, float("nan"), 0.0, 0.0))
print(f"| kernel (batch N={n}) | GFLOP | us | TFLOP/s | of measured peak ({peak:.0f}) |\n|---|---|---|---|---|")
for r in rows:
    print(f"| {r[0]} | {r[1]:.2f} | {r[2]:.1f} | {r[3]:.0f} | {r[4]:.2f} |")
tot_f = sum(r[1] for r in rows); tot_t = sum(r[2] for r in rows if r[2] == r[2]) or 1.0
print(f"| all | {tot_f:.1f} | {tot_t:.0f} | {tot_f / tot_t * 1e3:.0f} | {tot_f / tot_t * 1e3 / peak:.2f} |")
print(f"\n| skinny layer (batch N={n}) | GFLOP | activation MB | SIMT us | tensor-core us |\n|---|---|---|---|---|")
for r in edge_rows:
    print(f"| {r[0]} | {r[1]:.2f} | {r[2]:.1f} | {r[3]:.1f} | {r[4]:.1f} |")
ctx.close()
