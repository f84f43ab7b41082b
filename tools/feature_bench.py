"""Cost of one library feature on bench.py's workloads (bf16, CUDA-graph steps, one GPU), every feature under one protocol.

    python tools/feature_bench.py FEATURE [--configs c5,c2] [--steps N] [--rounds R] [--out OUT.json]

FEATURE is a key of FEATURES below, which also holds each feature's default configs, steps and rounds.  Every case is a bench.py config as
bench.make_gan builds it (seeds 666 / 667, xent_clip_eps 0, D with bn_groups 2, bf16, CUDA graph; data bench.synthetic(cfg, n, 666)), as it
is or in a variant: other builder arguments or updaters in the specs, a setting on both built nets, or other labels.
  1. runs: `--rounds` rounds; each round builds every case in turn, times `--steps` steps with bench.timed_resident_steps (10 warm-up steps,
     L2 flushed before each step, CUDA events per step, as bench.py times its configurations), counts kernel launches and SIMT GEMM calls over
     5 steps of their own, records the losses and closes the nets.  A row holds the mean and the median ms per step, so round means and the
     range of round medians both read off it.
  2. step_kernels: the feature's kernels inside the step, torch.profiler (CUDA activities) over 50 replayed steps after 10 warm-up steps, in a
     run of their own per case, with their algorithmic bytes (the byte models below) over kernel time as a fraction of the H100 SXM data-sheet
     3.35 TB/s.  The operands were mostly written moments earlier, so part of them comes from L2: the fractions are not measured HBM rates.
  3. kernels: the feature's kernels alone through the test hooks at the sizes its workloads run them.
The card's name, power limit and max SM clock are read in the same process as the timings.  Prints one JSON object; --out writes it too."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

import bench
import gan_deeplearning4j_b200 as b
from gan_deeplearning4j_b200 import engine, models as m

# the data sheet's figure, not bench.load_peaks(): the fractions keep one denominator whether or not MEASURED_PEAKS.json exists
HBM_BYTES_PER_S = 3.35e12
LAUNCH_STEPS = 5


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                              check=True).stdout.strip()
    except Exception as e:          # the numbers are still taken; the card line says why it is missing
        return f"unavailable: {e}"


def fraction(nbytes, us):
    return nbytes / (us * 1e-6) / HBM_BYTES_PER_S if us else None


def kernel_us(prof, name):
    """Device time (µs) of each CUDA kernel event whose name contains `name`."""
    return [ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            for ev in prof.events() if name in ev.name and ev.device_type == torch.autograd.DeviceType.CUDA]


def build(ctx, cfg_name, variant):
    """(n, G, D, gan) as bench.make_gan builds them, with the variant's builder arguments ("g", "d"), its change to each spec list ("swap"),
    its setting on each built net ("hook") and its labels y_real, y_fake, y_gen ("labels") in place of bench.synthetic's."""
    cfg = bench.CONFIGS[cfg_name]
    g, d, n = variant.get("g", {}), variant.get("d", {}), cfg["batch"]
    if cfg.get("mlp"):
        gs, ds, gin, din = m.mlp_generator(cfg["z"], cfg["hidden"], cfg["d"], **g), m.mlp_discriminator(cfg["d"], cfg["hidden"], **d), (cfg["z"],), (cfg["d"],)
    else:
        gs, ds = m.dcgan_generator(cfg["size"], cfg["z"], cfg["nf"], cfg["nc"], **g), m.dcgan_discriminator(cfg["size"], cfg["nf"], cfg["nc"], **d)
        gin, din = (cfg["z"],), (cfg["nc"], cfg["size"], cfg["size"])
    swap = variant.get("swap", list)
    G = b.Net(ctx, swap(gs), gin, max_batch=n, precision=b.BF16, xent_clip_eps=0.0, seed=666)
    D = b.Net(ctx, variant.get("d_swap", list)(swap(ds)), din, max_batch=2 * n, precision=b.BF16, xent_clip_eps=0.0, bn_groups=2, seed=667)
    gan = b.Gan(G, D, fake_bn_train=False, use_cuda_graph=True)
    if "hook" in variant:
        variant["hook"](G); variant["hook"](D)
    if "gan_hook" in variant:
        variant["gan_hook"](gan, D, n)
    data = bench.synthetic(cfg, n, 666)
    if "labels" in variant:
        data = data[:3] + [np.full((n, 1), v, np.float32) for v in variant["labels"]]
    gan.upload(*data)
    return n, G, D, gan


def label(cfg_name, variant):
    return f"{cfg_name}+{variant['name']}" if "name" in variant else cfg_name


def step_rounds(ctx, cases, steps, rounds):
    runs = []
    for r in range(rounds):
        for cfg_name, v in cases:
            n, G, D, gan = build(ctx, cfg_name, v)
            ms = bench.timed_resident_steps(ctx, gan, n, steps, 10, ctx.sync)
            simt = lambda: G.simt_gemm_calls() + D.simt_gemm_calls()
            l0, s0 = ctx.launch_count(), simt()          # launches of graph-replayed steps only, counted around steps of their own
            for _ in range(LAUNCH_STEPS):
                gan.step_resident(n)
            ctx.sync()
            runs.append({"config": label(cfg_name, v), "round": r, "ms_per_step": float(np.mean(ms)), "median_ms_per_step": float(np.median(ms)),
                         "samples_per_s": n * len(ms) / (sum(ms) * 1e-3), "launches_per_step": (ctx.launch_count() - l0) / LAUNCH_STEPS,
                         "simt_calls_per_step": (simt() - s0) / LAUNCH_STEPS, "losses": [float(x) for x in gan.losses()]})
            gan.close(); G.close(); D.close()
    return runs


def in_step_kernels(ctx, gan, n, names, steps=50):
    """{kernel name: launches and µs per step} over `steps` graph-replayed steps under torch.profiler, after 10 warm-up steps."""
    for _ in range(10):
        gan.step_resident(n)
    ctx.sync()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            gan.step_resident(n)
        ctx.sync()
    out = {}
    for name in names:
        t = kernel_us(prof, name)
        out[name] = {"launches_per_step": len(t) / steps, "us_per_step": sum(t) / steps}
    return out


def step_kernel_rows(ctx, cases):
    """The in-step kernels of every case that names them, with what its byte model ("model": cfg, G, D, n -> fields) adds: "bytes_per_step"
    over all the named kernels, or "kernel_bytes_per_step" per kernel."""
    rows = {}
    for cfg_name, v in cases:
        if "kernels" not in v:
            continue
        n, G, D, gan = build(ctx, cfg_name, v)
        row = v["model"](bench.CONFIGS[cfg_name], G, D, n) if "model" in v else {}
        row["kernels"] = ks = in_step_kernels(ctx, gan, n, v["kernels"])
        row["launches_per_step"] = sum(k["launches_per_step"] for k in ks.values())
        row["us_per_step"] = sum(k["us_per_step"] for k in ks.values())
        if "bytes_per_step" in row:
            row["fraction_of_3_35_TBps"] = fraction(row["bytes_per_step"], row["us_per_step"])
        for name, nbytes in row.get("kernel_bytes_per_step", {}).items():
            ks[name]["fraction_of_3_35_TBps"] = fraction(nbytes, ks[name]["us_per_step"])
        rows[label(cfg_name, v)] = row
        gan.close(); G.close(); D.close()
    return rows


def hook_kernel(ctx, call, names, reps, flush, stat):
    """A test-hook call once to warm up (its result is returned), then `reps` times under torch.profiler, L2 flushed before each call if
    `flush`; {kernel name: stat (np.mean / np.median) of its µs per launch, and its launches}."""
    first = call()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            if flush:
                ctx.flush_l2()
            call()
        ctx.sync()
    out = {}
    for name in names:
        t = kernel_us(prof, name)
        out[name] = {"us": float(stat(t)) if t else None, "calls": len(t)}
    return first, out


# ---------------------------------------------------------------- activation: ReLU / LeakyReLU replaced by ELU, then SELU
def ext_bytes_per_step(net, spec_list, fwd_rows, bwd_rows):
    """Algorithmic bytes of the act_ext kernels of one net per step: its layers of codes 5-16, forwards over fwd_rows rows in all, backwards over
    bwd_rows (bf16: 4 B / element forward, 6 B / element backward)."""
    elems = sum(net.layer_output_size(i) for i, s in enumerate(spec_list) if engine.ACTS[s.get("activation", "identity")] >= 5)
    return elems * (4 * fwd_rows + 6 * bwd_rows)


def activation_model(cfg, G, D, n):
    # per step: G forward on z_d and on z_g (N rows each), G backward (N); D forward on real|fake (2N) and on G's output (N), D backward on both
    return {"bytes_per_step": ext_bytes_per_step(G, G.specs, 2 * n, n) + ext_bytes_per_step(D, D.specs, 3 * n, 3 * n)}


# ---------------------------------------------------------------- constraint: MaxNorm(1.0) per output unit on every W of G and D
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


def constraint_model(cfg, G, D, n):
    """Bytes per constrained parameter: 10 on the one-pass path (read 4, write 4, bf16 copy 2), 14 on the two-launch path (norm read 4, scale
    read 4 + write 4, bf16 copy 2); the packed pixel-shuffle copy (2 B for G's last W only) and the per-group partials are left out.  Which
    tensor takes which path is the rule stated at b2g_constraint in include/b200gan.h."""
    tensors = {sp["name"]: path(sp) for net in (G, D) for sp in with_n_in(net)}
    return {"paths": {k: {"path": p, "params": c} for k, (p, c) in tensors.items()}, "constrained_params": sum(c for _, c in tensors.values()),
            "bytes_per_step": sum((10 if p == "one-pass" else 14) * c for p, c in tensors.values())}


# ---------------------------------------------------------------- dropout: C5 with DropoutLayer(0.5) after each hidden LeakyReLU of D
def dropout_model(cfg, G, D, n):
    """Bytes per masked element, bf16: forward reads x (2 B), writes y (2 B) and one mask bit; backward reads dy (2 B) and the bit, writes dx
    (2 B).  Per step D runs them on its 2N-row pass and on the generator step's N-row pass, over two hidden layers."""
    elems = 2 * (2 * n + n) * cfg["hidden"]          # masked elements per step, forward (the backward handles the same)
    each_way = elems * (2 + 2 + 1 / 8)
    return {"masked_elements_per_step": elems, "kernel_bytes_per_step": {"dropout_fwd_kernel": each_way, "dropout_bwd_kernel": each_way}}


# ---------------------------------------------------------------- noise: instance noise on D's input (C5, C2); GaussianDropout(0.5) or
# AlphaDropout(0.9) after each hidden LeakyReLU of D (C5), beside C5's DropoutLayer(0.5) in the same session
def after_lrelu(make):
    def swap(specs):
        out = []
        for s in specs:
            out.append(s)
            if s.get("activation") == "lrelu":
                out.append(make(s["name"] + "_noise"))
        return out
    return swap


def noise_model(fwd_kernel, fwd_bytes, bwd_kernel, bwd_bytes):
    """Algorithmic bytes per element of D's DropoutLayers, bf16: GaussianNoise reads x and writes y (4 B) and has no backward;
    GaussianDropout 4 B each way (its backward draws m again); AlphaDropout 4 B and one mask bit each way (bern_fwd_kernel, mask_bwd_kernel).  Per step D runs them on its 2N-row
    pass and on the generator step's N-row pass.  GaussianDropout's forward and backward are one kernel (gauss_kernel)."""
    def model(cfg, G, D, n):
        elems = 3 * n * sum(D.layer_output_size(i) for i, s in enumerate(D.specs) if s["type"] == "dropout")
        kb = {fwd_kernel: elems * fwd_bytes}
        if bwd_bytes:
            kb[bwd_kernel] = kb.get(bwd_kernel, 0) + elems * bwd_bytes
        return {"noisy_elements_per_step": elems, "kernel_bytes_per_step": kb}
    return model


# ---------------------------------------------------------------- weightnoise: DropConnect(0.9) on every GEMM layer of D (C5, C2); on C5 also
# WeightNoise(Normal(0, 0.01)) on every layer of G
def g_normal_noise(net):
    if net.specs[0]["name"].startswith("gen"):
        net.set_weight_noise(m.weight_noise(m.normal(0.0, 0.01)))


def weight_noise_model(cfg, G, D, n):
    """Bytes per noisy bf16 weight and draw: read the fp32 master (4 B), write the bf16 straight copy (2 B), and 2 B more for a layer with the
    packed pixel-shuffle copy (a 4x4 s2 p1 conv from or transposed conv onto <= 4 channels, 64k units: C2's D-first and G-last).  D draws in
    both of its passes per step, G in its one train-mode pass; biases are not perturbed."""
    def per_draw(net):
        tot = 0
        for sp in with_n_in(net):
            if sp.get("weight_noise") is None:
                continue
            k = sp.get("kernel", (1, 1)) if sp["type"] in ("conv2d", "deconv2d") else (1, 1)
            nw = sp["n_in"] * sp["n_out"] * k[0] * k[1]
            img, units = (sp["n_out"], sp["n_in"]) if sp["type"] == "deconv2d" else (sp["n_in"], sp["n_out"])
            packed = tuple(k) == (4, 4) and tuple(sp.get("stride", ())) == (2, 2) and tuple(sp.get("padding", ())) == (1, 1) and img <= 4 and units % 64 == 0
            tot += nw * (8 if packed else 6)
        return tot
    return {"bytes_per_draw_D": per_draw(D), "bytes_per_draw_G": per_draw(G), "bytes_per_step": 2 * per_draw(D) + per_draw(G)}


# ---------------------------------------------------------------- gradnorm: RenormalizeL2PerLayer on C5, ClipL2PerLayer(1.0) on C2
def gradnorm_model(cfg, G, D, n):
    """The norm kernel reads every gradient once, 4 B per parameter of G and D per step (it writes one double per 4096 parameters and one
    float per parameter tensor)."""
    params = G.num_params() + D.num_params()
    return {"params_G_plus_D": params, "bytes_per_step": 4 * params}


def gradnorm(mode):
    return dict(name=mode, hook=lambda net: net.set_gradient_normalization(mode, 1.0), kernels=("gradnorm_kernel",), model=gradnorm_model)


# ---------------------------------------------------------------- graph: residual C2, a U-Net fit and the vertex kernels
def unet_step(ctx, steps, weighted=False):
    """weighted: class weights (0.5, 2) and a per-pixel labels mask (a quarter of the pixels 0), as a segmentation run with void pixels has."""
    n, size = 128, 64
    net = b.Net(ctx, m.unet(size, 3, 2, 32, 2), (3, size, size), max_batch=n, precision=b.BF16)
    rng = np.random.default_rng(1)
    x = rng.uniform(-1, 1, (n, 3, size, size)).astype(np.float32)
    lab = rng.integers(0, 2, (n, size, size))
    y = np.ascontiguousarray(np.moveaxis(np.eye(2, dtype=np.float32)[lab], -1, 1))
    mask = (rng.uniform(0, 1, (n, 1, size, size)) > 0.25).astype(np.float32) if weighted else None
    if weighted:
        net.set_loss_weights([0.5, 2.0])
    for _ in range(3):
        net.fit(x, y, mask=mask)
    s0, l0 = net.simt_gemm_calls(), ctx.launch_count()
    t0 = time.perf_counter()
    for _ in range(steps):
        net.fit(x, y, mask=mask)         # returns after a device synchronise
    ms = (time.perf_counter() - t0) * 1e3 / steps
    res = {"ms_per_fit_incl_host_copies": round(ms, 3), "simt_calls_per_fit": (net.simt_gemm_calls() - s0) / steps,
           "launches_per_fit": (ctx.launch_count() - l0) / steps}
    net.close()
    return res


def vertex_kernels(ctx):
    """The vertex kernels alone through b2g_test_ew, 5 calls each, at the sizes the residual C2 step and the U-Net run them."""
    # (label, op, test_ew arguments, input sizes, kernel name, algorithmic bytes per call in bf16)
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
    for name, op, kw, n0, n1, kname, byts in cases:
        a = rng.uniform(-1, 1, n0).astype(np.float32)
        bb = rng.uniform(-1, 1, n1).astype(np.float32) if n1 else None
        extra = {"act": "add"} if op.startswith("vertex") else {}
        _, t = hook_kernel(ctx, lambda: b.test_ew(ctx, b.BF16, op, a, bb, (0, 0, 0), **extra, **kw), (kname,), 5, False, np.mean)
        res[name] = dict(t[kname], kernel=kname, algorithmic_bytes=byts, fraction_of_3_35_TBps=fraction(byts, t[kname]["us"]))
    return res


# ---------------------------------------------------------------- loss: D on XENT, MSE, Hinge and Wasserstein
def loss_fit_output(ctx):
    """The loss kernel alone on a [8192 x 256] MSE fit output (b2g_test_ew, bf16, identity and tanh), 50 calls, at 8 B per element (z and dz
    2 B each, the fp32 labels 4 B).  The operands were just uploaded, so part of them may come from L2: the fraction is an upper bound on the
    HBM rate, not a roofline."""
    rows, n_out = 8192, 256
    rng = np.random.default_rng(0)
    z = rng.standard_normal((rows, n_out)).astype(np.float32); y = rng.uniform(-1, 1, (rows, n_out)).astype(np.float32)
    res = {}
    for act in ("identity", "tanh"):
        call = lambda: b.test_ew(ctx, b.BF16, "loss", z, y, (z.size, 1, 0), act=act, loss="mse", rows=rows, cols=n_out, groups=1)
        _, t = hook_kernel(ctx, call, ("loss_kernel",), 50, False, np.mean)
        res[f"mse+{act}"] = dict(t["loss_kernel"], shape=[rows, n_out], bytes=rows * n_out * 8, fraction_of_3_35_TBps=fraction(rows * n_out * 8, t["loss_kernel"]["us"]))
    return res


# MSE with least-squares GAN labels 1 / 0 / 1, Hinge and Wasserstein with +1 / -1 / +1
LOSS_LABELS = {"mse": (1.0, 0.0, 1.0), "hinge": (1.0, -1.0, 1.0), "wasserstein": (1.0, -1.0, 1.0)}


# ---------------------------------------------------------------- patchgan: dcgan_discriminator(patch=True), its head conv, CnnLossLayer
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


def head_conv(ctx, configs, steps):
    """The head conv at the patch shapes of the D step through b2g_test_conv_ex (CUDA events over 20 launches, warm L2): the SIMT route (impl 0)
    against the few-output kernels (impl 5)."""
    out = {}
    for c in configs:
        g = head_geom(bench.CONFIGS[c], 2 * bench.CONFIGS[c]["batch"])
        out[c + "_patch (D step, 2N)"] = {"geom": g, **head_times(ctx, g)}
    return {"head_conv": out}


def cnn_loss_kernels(ctx):
    """The CnnLossLayer kernels alone through b2g_test_ew, 5 calls each; algorithmic bytes = z + dz (2 B each in bf16) + labels (4 B) per element."""
    cases = {"cnn_xent C2 patch D step (2 x 128 x 16)": ("cnn_xent", 2, 128 * 16, 1),
             "cnn_xent 2 x 64 x 64 x 64 map": ("cnn_xent", 2, 64 * 64 * 64, 1),
             "cnn_softmax_xent 16 x 128 x 128 pixels, C = 21": ("cnn_softmax_xent", 1, 16 * 128 * 128, 21)}
    res = {}
    for name, (op, groups, rows, c) in cases.items():
        n = groups * rows * c
        rng = np.random.default_rng(2)
        z, y = rng.uniform(-3, 3, n).astype(np.float32), rng.uniform(0, 1, n).astype(np.float32)
        _, t = hook_kernel(ctx, lambda: b.test_ew(ctx, b.BF16, op, z, y, (0, 0, 0), rows=rows, cols=c, groups=groups), (f"{op}_kernel",), 5, False, np.mean)
        byts = n * (2 + 2 + 4)
        res[name] = dict(t[f"{op}_kernel"], algorithmic_bytes=byts, fraction_of_3_35_TBps=fraction(byts, t[f"{op}_kernel"]["us"]))
    return res


# ---------------------------------------------------------------- lossmask: per-output loss weights and labels masks
def patch_masks(gan, D, n):
    """Per-patch labels masks on the C2 patch step: the border patches of the 4 x 4 map masked out, the inner ones 1."""
    mk = np.zeros((n, 1, 4, 4), np.float32)
    mk[:, :, 1:3, 1:3] = 1
    gan.set_label_masks(mk, mk, mk)


def loss_mask_kernels(ctx):
    """The MCXENT and XENT CnnLossLayer kernels at a segmentation size, 16 x 128 x 128 pixels x 21 classes, unweighted and with class weights and
    a per-pixel mask: a net of one identity ActivationLayer into the CnnLossLayer, fit 5 times under torch.profiler.  Algorithmic bytes per
    element: z + dz (2 B each, bf16) + labels (4 B); the mask adds 4 B per pixel and the weights are left out."""
    n, c, hw = 16, 21, 128
    rng = np.random.default_rng(3)
    x = rng.uniform(-3, 3, (n, c, hw, hw)).astype(np.float32)
    lab = rng.integers(0, c, (n, hw, hw))
    y1 = np.ascontiguousarray(np.moveaxis(np.eye(c, dtype=np.float32)[lab], -1, 1))
    mask = (rng.uniform(0, 1, (n, 1, hw, hw)) > 0.25).astype(np.float32)
    res = {}
    for loss, kern in (("mcxent", "cnn_softmax_xent_kernel"), ("xent", "cnn_xent_kernel")):
        for weighted in (False, True):
            net = b.Net(ctx, [{"type": "activation", "name": "a", "activation": "identity"}, m.cnn_loss(loss, name="cl")], (c, hw, hw), max_batch=n,
                        precision=b.BF16)
            if weighted:
                net.set_loss_weights(np.linspace(0.5, 2.0, c))
            for _ in range(2):
                net.fit(x, y1, mask=mask if weighted else None)
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    net.fit(x, y1, mask=mask if weighted else None)
            t = kernel_us(prof, kern)
            us = float(np.mean(t)) if t else None
            byts = n * hw * hw * (c * (2 + 2 + 4) + (4 if weighted else 0))
            res[f"{kern} {'weights + mask' if weighted else 'plain'}"] = {"us": us, "launches_per_fit": len(t) / 5, "algorithmic_bytes": byts,
                                                                          "fraction_of_3_35_TBps": fraction(byts, us)}
            net.close()
    return res


# ---------------------------------------------------------------- pooling: C2 with a global SUM / AVG head, and the pooling kernels
TS = 2                          # bf16 bytes
SUB_SHAPES = [(256, 32, 32, 64), (256, 16, 16, 128)]
GLOBAL_SHAPES = [(256, 4, 4, 512), (32, 64, 64, 128)]


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


def pool_case(ctx, op, kind, shape):
    """One pooling layer's kernels through b2g_test_pool (NHWC bf16), median of 5 calls with L2 flushed before each.  The hook writes the inputs
    on the device right before the forward, so part of them may still sit in L2."""
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
    (_, info), t = hook_kernel(ctx, call, (f"{op}_fwd_kernel", f"{op}_bwd_kernel"), 5, True, np.median)
    out = {"op": op, "kind": kind, "shape_nhwc": list(shape), "kernels": info["kernel"], "global_splits": info["splits"] if op == "global_pool" else None}
    for d, nbytes in (("fwd", fb), ("bwd", bb)):
        k = t[f"{op}_{d}_kernel"]
        out[d] = dict(k, bytes=nbytes, fraction_of_3_35_TBps=fraction(nbytes, k["us"]))
    return out


def pooling_kernels(ctx):
    return ([pool_case(ctx, "pool2d", kind, s) for s in SUB_SHAPES for kind in ("avg", "pnorm")] +
            [pool_case(ctx, "global_pool", kind, s) for s in GLOBAL_SHAPES for kind in ("max", "avg", "pnorm")])


# ---------------------------------------------------------------- schedule: ExponentialSchedule(ITERATION, lr, 0.9999) on every layer
def schedule(net):
    lr = net.learning_rate(next(s["name"] for s in net.specs if s.get("updater")))
    net.set_lr_schedule(m.exponential_schedule(lr, 0.9999))


def params_model(cfg, G, D, n):
    return {"params_G_plus_D": G.num_params() + D.num_params()}


UPDATER = ("updater_kernel",)


# ---------------------------------------------------------------- updater: every layer of G and D on one updater kind
# per-kind traffic (include/b200gan.h, DESIGN.md 3), each + 2 B for the bf16 operand copy
BYTES_PER_PARAM = {"adam": 28, "nesterovs": 20, "adagrad": 20, "adamax": 28, "nadam": 28, "amsgrad": 36, "adadelta": 28}


def with_kind(specs, kind):
    """Every updater of the specs replaced by `kind` at the layer's Adam learning rate (AdaDelta: DL4J's defaults, no learning rate)."""
    out = []
    for s in specs:
        s = dict(s)
        if s.get("updater"):
            lr = s["updater"]["lr"]
            s["updater"] = m.adadelta() if kind == "adadelta" else m.nesterovs(lr) if kind == "nesterovs" else getattr(m, kind)(lr)
        out.append(s)
    return out


def updater(kind):
    def model(cfg, G, D, n):
        params = G.num_params() + D.num_params()
        return {"params_G_plus_D": params, "bytes_per_step": params * (BYTES_PER_PARAM[kind] + 2)}
    return dict(name=kind, swap=lambda s: with_kind(s, kind), kernels=UPDATER, model=model)


# ---------------------------------------------------------------- regularization: the reference's l2 1e-4 on every W, against l1, l2, l1Bias
# and l2Bias on every layer (the same one updater pass; the score sums are not part of the step)
def regularize(**coefs):
    return lambda net: net.set_regularization(**coefs)


# ---------------------------------------------------------------- weightinit: b2g_net_init_weights over bench.py's nets
INIT_SCHEMES = (("distribution_normal_0.02", m.weight_init("distribution", m.normal(0, 0.02))), ("xavier", m.weight_init("xavier")),
                ("xavier_uniform", m.weight_init("xavier_uniform")), ("var_scaling_normal_fan_avg", m.weight_init("var_scaling_normal_fan_avg")))


def init_weights_times(ctx, configs):
    """Per config, on G and D as bench.make_gan builds them (BF16): the host time of b2g_net_create, and for a few schemes one
    b2g_net_init_weights call (layer NULL) on each net, measured two ways after one warm-up pair of calls:
      call_ms        CUDA events on the library stream around the two calls, median of 5: what a caller waits, host-side checks, one launch
                     per layer and the closing stream synchronisation included -- a latency, not a kernel time;
      kernel_us      torch.profiler device time of the weight_init_kernel launches of one pair of calls (mean of 5), and refresh_us that of the
                     bf16 operand refresh (cast_f32_to_bf16_kernel, pack_deconv_ps_kernel) that follows them.
    hbm_fraction: the kernel's algorithmic bytes, 4 B written per parameter (BatchNorm's few included), over kernel_us, as a fraction of the
    3.35 TB/s data sheet."""
    out = {}
    for cfg_name in configs:
        cfg = bench.CONFIGS[cfg_name]
        t0 = time.perf_counter()
        G, D, gan = bench.make_gan(b, ctx, cfg, cfg["batch"])
        create_ms = (time.perf_counter() - t0) * 1e3
        gan.close()
        params = G.num_params() + D.num_params()
        rows = {}
        for name, wi in INIT_SCHEMES:
            G.init_weights(wi); D.init_weights(wi)          # warm-up
            ms = []
            for _ in range(5):
                ctx.sync(); ctx.timer_start()
                G.init_weights(wi); D.init_weights(wi)
                ms.append(ctx.timer_stop_ms())
            ctx.sync()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    G.init_weights(wi); D.init_weights(wi)
                ctx.sync()
            k = kernel_us(prof, "weight_init_kernel")
            refresh = sum(kernel_us(prof, "cast_f32_to_bf16_kernel")) + sum(kernel_us(prof, "pack_deconv_ps_kernel"))
            kus = sum(k) / 5
            rows[name] = {"call_ms": float(np.median(ms)), "kernel_launches": len(k) / 5, "kernel_us": kus, "refresh_us": refresh / 5,
                          "hbm_fraction": fraction(params * 4, kus)}
        out[cfg_name] = {"params": params, "net_create_host_ms": create_ms, "init_weights": rows}
        G.close(); D.close()
    return out


# ---------------------------------------------------------------- prelu: C2 with activation="prelu" in both nets (PReLULayers shared over H
# and W in place of the ActivationLayers, D's first conv identity + PReLU) against plain C2
def prelu_model(cfg, G, D, n):
    """Algorithmic bytes of the PReLU kernels per step, bf16: the forward reads x and writes y (4 B / element); the backward reads x and dy and
    writes dx (6 B / element), and in a trainable pass also its fp32 slope partials (4 B per row group and row element; the reduce-list job
    that folds them is not counted).  G runs its layers forward on z_d and z_g (N rows each) and backward on N; D forward on real|fake (2N)
    and on G's output (N), backward on both.  The fp32 slopes (one per channel) are left out."""
    def elems(net):
        return [net.layer_output_size(i) for i, s in enumerate(net.specs) if s["type"] == "prelu"]
    def parts(net, rows):
        return sum(4 * engine.prelu_groups(rows, e) * e for e in elems(net))
    g, d = sum(elems(G)), sum(elems(D))
    return {"prelu_elements_per_row_G": g, "prelu_elements_per_row_D": d,
            "kernel_bytes_per_step": {"prelu_fwd_kernel": 4 * (2 * n * g + 3 * n * d),
                                      "prelu_bwd_kernel": 6 * (n * g + 3 * n * d) + parts(G, n) + parts(D, 2 * n)}}


ACT_EXT = ("act_ext_fwd_kernel", "act_ext_bwd_kernel")
CONSTRAINT = ("constraint_onepass_kernel", "constraint_norm_kernel", "constraint_scale_kernel")
# each feature: default configs, steps, rounds; its variants ("only": the configs it runs on; "kernels": the in-step kernels to profile);
# "kernels": its isolated-kernel section; "extras": further sections (ctx, configs, steps -> {key: ...})
FEATURES = {
    "activation": dict(configs="c5,c2", variants=[dict(name="base")] + [
        dict(name=k, g=dict(activation=k), d=dict(activation=k), kernels=ACT_EXT, model=activation_model) for k in ("elu", "selu")]),
    "constraint": dict(configs="c5,c2", variants=[{}, dict(name="maxnorm", hook=constrain, kernels=CONSTRAINT, model=constraint_model)]),
    "dropout": dict(configs="c5", variants=[{}, dict(name="dropout", d=dict(dropout=0.5), kernels=("dropout_fwd_kernel", "dropout_bwd_kernel"),
                                                     model=dropout_model)]),
    "noise": dict(configs="c5,c2", variants=[
        {}, dict(name="instance_noise", d=dict(instance_noise=0.1), kernels=("gauss_kernel",), model=noise_model("gauss_kernel", 4, None, 0)),
        dict(name="gaussian_dropout", only=("c5",), d_swap=after_lrelu(lambda nm: m.gaussian_dropout(0.5, nm)), kernels=("gauss_kernel",),
             model=noise_model("gauss_kernel", 4, "gauss_kernel", 4)),
        dict(name="alpha_dropout", only=("c5",), d_swap=after_lrelu(lambda nm: m.alpha_dropout(0.9, nm)), kernels=("bern_fwd_kernel", "mask_bwd_kernel"),
             model=noise_model("bern_fwd_kernel", 4.125, "mask_bwd_kernel", 4.125)),
        dict(name="dropout", only=("c5",), d=dict(dropout=0.5), kernels=("dropout_fwd_kernel", "dropout_bwd_kernel"), model=dropout_model)]),
    "gradnorm": dict(configs="c5,c2", variants=[{}, dict(gradnorm("renormalize_l2_per_layer"), only=("c5",)),
                                                dict(gradnorm("clip_l2_per_layer"), only=("c2",))]),
    "graph": dict(configs="c2", steps=50, variants=[{}, dict(name="residual", g=dict(residual=True), d=dict(residual=True))],
                  kernels=vertex_kernels, extras=lambda ctx, configs, steps: {"unet": unet_step(ctx, max(5, steps // 5))}),
    "loss": dict(configs="c5,c2", variants=[dict(name="xent", kernels=("xent_kernel",))] + [
        dict(name=k, d=dict(loss=k), labels=lab, kernels=("loss_kernel",)) for k, lab in LOSS_LABELS.items()], kernels=loss_fit_output),
    "lossmask": dict(configs="c2", steps=50, variants=[dict(name="patch", d=dict(patch=True), kernels=("cnn_xent_kernel",)),
                                                       dict(name="patch+mask", d=dict(patch=True), gan_hook=patch_masks, kernels=("cnn_xent_kernel",))],
                     kernels=loss_mask_kernels,
                     extras=lambda ctx, configs, steps: {"unet": unet_step(ctx, max(5, steps // 5)),
                                                          "unet_weights_mask": unet_step(ctx, max(5, steps // 5), weighted=True)}),
    "patchgan": dict(configs="c2,c4", steps=50, variants=[{}, dict(name="patch", d=dict(patch=True))], kernels=cnn_loss_kernels, extras=head_conv),
    "pooling": dict(configs="c2", variants=[dict(name="base"), dict(name="sum", d=dict(global_pooling="sum")),
                                            dict(name="avg", d=dict(global_pooling="avg"))], kernels=pooling_kernels),
    "prelu": dict(configs="c2", variants=[{}, dict(name="prelu", g=dict(activation="prelu"), d=dict(activation="prelu"),
                                                   kernels=("prelu_fwd_kernel", "prelu_bwd_kernel", "reduce_multi_kernel"), model=prelu_model)]),
    "regularization": dict(configs="c5,c2", variants=[
        dict(name="l2", hook=regularize(l2=1e-4), kernels=UPDATER, model=params_model),
        dict(name="l1+l2+l1bias+l2bias", hook=regularize(l1=1e-4, l2=1e-4, l1_bias=1e-4, l2_bias=1e-4), kernels=UPDATER, model=params_model)]),
    "schedule": dict(configs="c5,c2", variants=[dict(kernels=UPDATER, model=params_model),
                                                dict(name="exponential_schedule", hook=schedule, kernels=UPDATER, model=params_model)]),
    "updater": dict(configs="c5,c2", variants=[updater(k) for k in ("adam", "nesterovs", "adagrad", "adamax", "nadam", "amsgrad", "adadelta")]),
    "weightinit": dict(configs="c4,c2", variants=[], extras=lambda ctx, configs, steps: {"init_weights": init_weights_times(ctx, configs)}),
    "weightnoise": dict(configs="c5,c2", variants=[
        {}, dict(name="dropconnect", d=dict(drop_connect=0.9), kernels=("weight_noise_kernel",), model=weight_noise_model),
        dict(name="dropconnect+g_normal", only=("c5",), d=dict(drop_connect=0.9), hook=g_normal_noise, kernels=("weight_noise_kernel",),
             model=weight_noise_model)]),
}


def main():
    ap = argparse.ArgumentParser(description="Cost of one library feature on bench.py's workloads (see the module docstring).")
    ap.add_argument("feature", choices=sorted(FEATURES))
    ap.add_argument("--configs", default=None, help="comma-separated bench.py configs (default: the feature's)")
    ap.add_argument("--steps", type=int, default=None, help="timed steps per case and round (default: 50 for graph and patchgan, else 100)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    a = ap.parse_args()
    f = FEATURES[a.feature]
    configs = (a.configs or f["configs"]).split(",")
    steps = a.steps or f.get("steps", 100)
    cases = [(c, v) for c in configs for v in f["variants"] if c in v.get("only", (c,))]
    ctx = b.Context(0)
    res = {"card": card(), "feature": a.feature, "steps": steps, "runs": step_rounds(ctx, cases, steps, a.rounds),
           "step_kernels": step_kernel_rows(ctx, cases), "kernels": f["kernels"](ctx) if "kernels" in f else {}}
    if "extras" in f:
        res.update(f["extras"](ctx, configs, steps))
    ctx.close()
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
