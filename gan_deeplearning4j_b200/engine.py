"""Host-side mirror of the C-ABI objects: Context (b2g_ctx), Net (b2g_net ~ ComputationGraph), Gan (b2g_gan).

Layer specs are plain dicts (see models.py); `layer_desc` turns one into the C struct the Java facade's layer
builders fill (ConvolutionLayer.Builder(kH,kW).stride().padding().nIn().nOut() ... J:135-140).
All tensors cross as NumPy fp32 arrays in DL4J layouts (NCHW / [N,F]; parameters in flattened-view order).
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence

import numpy as np

from . import _lib
from ._lib import GanConfig, LayerDesc, NetConfig, check

LAYER_TYPES = {"conv2d": 0, "deconv2d": 1, "batchnorm": 2, "dense": 3, "activation": 4, "maxpool": 5, "upsample2d": 6,
               "output": 7, "loss": 8, "ff_to_cnn": 9, "cnn_to_ff": 10, "dropout": 11}
ACTS = {"identity": 0, "tanh": 1, "sigmoid": 2, "relu": 3, "lrelu": 4}
UPDATERS = {"sgd": 0, "rmsprop": 1, "adam": 2, "noop": 3}
# DL4J GradientNormalization -> b2g_gradient_normalization (DL4J's ordinals).  ClipElementWiseAbsoluteValue is the `grad_clip` argument of Net.
GRADIENT_NORMALIZATIONS = {"none": 0, "renormalize_l2_per_layer": 1, "renormalize_l2_per_param_type": 2, "clip_l2_per_layer": 4,
                           "clip_l2_per_param_type": 5}
FP32, BF16 = 0, 1


def _fp(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _f32(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.float32)


def layer_desc(spec: Dict) -> LayerDesc:
    d = LayerDesc()
    d.type = LAYER_TYPES[spec["type"]]
    d.name = spec.get("name", "").encode()[:63]
    d.n_in, d.n_out = spec.get("n_in", 0), spec.get("n_out", 0)
    k, s, p = spec.get("kernel", (1, 1)), spec.get("stride", (1, 1)), spec.get("padding", (0, 0))
    if spec["type"] == "upsample2d":
        k = (spec.get("size", 2), spec.get("size", 2))
    d.k_h, d.k_w, d.s_h, d.s_w, d.p_h, d.p_w = k[0], k[1], s[0], s[1], p[0], p[1]
    d.has_bias = 1 if spec.get("has_bias", True) else 0
    d.act = ACTS[spec.get("activation", "identity")]
    d.act_alpha = spec.get("alpha", 0.01)
    if spec["type"] == "dropout":       # DropoutLayer.Builder(p): p = retain probability, carried in act_alpha
        d.act_alpha = spec["p"]
    u = spec.get("updater") or {"kind": "sgd", "lr": 0.0}
    d.updater = UPDATERS[u["kind"]]
    d.lr = u.get("lr", 0.0)
    if u["kind"] == "rmsprop":          # RmsProp(learningRate, rmsDecay, epsilon)
        d.beta1, d.beta2, d.eps = u.get("rms_decay", 0.95), 0.0, u.get("eps", 1e-8)
    else:
        d.beta1, d.beta2, d.eps = u.get("beta1", 0.9), u.get("beta2", 0.999), u.get("eps", 1e-8)
    d.l2 = spec.get("l2", 0.0)
    d.bn_decay, d.bn_eps = spec.get("decay", 0.9), spec.get("eps", 1e-5)
    to = spec.get("to", (0, 0, 0))      # FeedForwardToCnnPreProcessor(h, w, c)
    d.pre_h, d.pre_w, d.pre_c = to
    d.loss = {"xent": 0, "mcxent": 1}[spec.get("loss", "xent")]
    d.frozen = 1 if spec.get("frozen", False) else 0
    return d


class Context:
    """b2g_ctx: one CUDA device + stream.  Replaces Nd4j backend selection / CudaEnvironment setup (J:103-115)."""

    def __init__(self, device: int = 0):
        self.lib = _lib.load()
        h = C.c_void_p()
        check(self.lib.b2g_ctx_create(device, C.byref(h)))
        self.h = h
        self.world, self.rank = 1, 0

    def sync(self):
        check(self.lib.b2g_sync(self.h))

    def timer_start(self):
        check(self.lib.b2g_timer_start(self.h))

    def timer_stop_ms(self) -> float:
        v = C.c_float()
        check(self.lib.b2g_timer_stop_ms(self.h, C.byref(v)))
        return v.value

    def flush_l2(self):
        check(self.lib.b2g_flush_l2(self.h))

    def launch_count(self) -> int:
        v = C.c_uint64()
        check(self.lib.b2g_launch_count(self.h, C.byref(v)))
        return v.value

    def device_info(self):
        sm, mj, mn, mem = C.c_int32(), C.c_int32(), C.c_int32(), C.c_uint64()
        check(self.lib.b2g_device_info(self.h, C.byref(sm), C.byref(mj), C.byref(mn), C.byref(mem)))
        return dict(sm_count=sm.value, cc=(mj.value, mn.value), mem_bytes=mem.value)

    def comm_init(self, world: int, rank: int, unique_id: bytes):
        buf = C.create_string_buffer(unique_id, 128)
        check(self.lib.b2g_ctx_comm_init(self.h, world, rank, C.cast(buf, C.c_void_p)))
        self.world, self.rank = world, rank

    def allreduce_test(self, a: np.ndarray) -> np.ndarray:
        a = _f32(a).copy()
        check(self.lib.b2g_ctx_allreduce_test(self.h, _fp(a), a.size))
        return a

    def close(self):
        if self.h:
            self.lib.b2g_ctx_destroy(self.h)
            self.h = None


def comm_unique_id() -> bytes:
    buf = C.create_string_buffer(128)
    check(_lib.load().b2g_comm_unique_id(C.cast(buf, C.c_void_p)))
    return buf.raw


class Net:
    """b2g_net: a chain-shaped ComputationGraph (init / output / fit / getLayer(..).getParam/setParam; J:166-170,420-510)."""

    def __init__(self, ctx: Context, specs: Sequence[Dict], input_shape, max_batch: int, precision: int = FP32,
                 grad_clip: float = 0.0, xent_clip_eps: float = 1e-5, bn_groups: int = 1, seed: int = 666,
                 gradient_normalization: str = "none", gradient_normalization_threshold: float = 1.0):
        self.ctx, self.lib, self.specs = ctx, ctx.lib, list(specs)
        c, h, w = input_shape if len(input_shape) == 3 else (input_shape[0], 1, 1)
        self.input_shape = tuple(input_shape)
        cfg = NetConfig(h, w, c, max_batch, precision, grad_clip, xent_clip_eps, bn_groups, seed)
        arr = (LayerDesc * len(specs))(*[layer_desc(s) for s in specs])
        hnd = C.c_void_p()
        check(self.lib.b2g_net_create(ctx.h, C.byref(cfg), arr, len(specs), C.byref(hnd)))
        self.h = hnd
        self.max_batch, self.precision = max_batch, precision
        n = C.c_int64()
        check(self.lib.b2g_net_num_params(self.h, C.byref(n)))
        self.n_params = n.value
        check(self.lib.b2g_net_output_size(self.h, C.byref(n)))
        self.out_elems = n.value
        if gradient_normalization != "none":
            try:
                self.set_gradient_normalization(gradient_normalization, gradient_normalization_threshold)
            except Exception:
                self.close()
                raise

    # --- parameters (DL4J flattened-view order) ---
    def num_params(self) -> int:
        return self.n_params

    def set_param(self, layer: str, name: str, value):
        v = _f32(value).ravel()
        check(self.lib.b2g_net_set_param(self.h, layer.encode(), name.encode(), _fp(v), v.size))

    def get_param(self, layer: str, name: str, size: int) -> np.ndarray:
        out = np.empty(size, np.float32)
        check(self.lib.b2g_net_get_param(self.h, layer.encode(), name.encode(), _fp(out), size))
        return out

    def params(self) -> np.ndarray:
        out = np.empty(self.n_params, np.float32)
        check(self.lib.b2g_net_get_params(self.h, _fp(out), out.size))
        return out

    def set_params(self, flat):
        v = _f32(flat).ravel()
        check(self.lib.b2g_net_set_params(self.h, _fp(v), v.size))

    def gradients(self) -> np.ndarray:
        out = np.empty(self.n_params, np.float32)
        check(self.lib.b2g_net_get_gradients(self.h, _fp(out), out.size))
        return out

    def updater_state(self) -> np.ndarray:
        out = np.empty(2 * self.n_params, np.float32)
        check(self.lib.b2g_net_get_updater_state(self.h, _fp(out), out.size))
        return out

    def set_updater_state(self, st):
        v = _f32(st).ravel()
        check(self.lib.b2g_net_set_updater_state(self.h, _fp(v), v.size))

    # --- checkpoint / resume (ModelSerializer.writeModel, J:606-618; serializer.py) ---
    def save(self, path, save_updater: bool = True):
        from . import serializer
        serializer.save_net(self, path, self.specs, self.input_shape, save_updater,
                            {"precision": "bf16" if self.precision == BF16 else "fp32", "max_batch": self.max_batch, "iteration": self.iteration(),
                             "dropout_pass": self.dropout_pass()})

    def restore(self, path, load_updater: bool = True):
        """Loads parameters (and updater state) of a checkpoint written by save() into this net (same architecture)."""
        from . import serializer
        return serializer.restore_into(self, path, load_updater)

    # --- execution ---
    def output(self, x, train: bool = False) -> np.ndarray:
        x = _f32(x)
        out = np.empty((x.shape[0], self.out_elems), np.float32)
        check(self.lib.b2g_net_output(self.h, _fp(x), x.shape[0], int(train), _fp(out)))
        return out

    def layer_output_size(self, layer: int) -> int:
        n = C.c_int64()
        check(self.lib.b2g_net_layer_output_size(self.h, layer, C.byref(n)))
        return n.value

    def activation(self, layer: int, batch: int) -> np.ndarray:
        out = np.empty((batch, self.layer_output_size(layer)), np.float32)
        check(self.lib.b2g_net_get_activation(self.h, layer, batch, _fp(out)))
        return out

    def compute_gradient_and_score(self, x, y) -> float:
        x, y = _f32(x), _f32(y)
        s = C.c_float()
        check(self.lib.b2g_net_compute_gradient_and_score(self.h, _fp(x), _fp(y), x.shape[0], C.byref(s)))
        return s.value

    def fit(self, x, y) -> float:
        x, y = _f32(x), _f32(y)
        s = C.c_float()
        check(self.lib.b2g_net_fit(self.h, _fp(x), _fp(y), x.shape[0], C.byref(s)))
        return s.value

    def set_gradient_normalization(self, mode: str, threshold: float = 1.0):
        """DL4J's GradientNormalization for every layer of the net, applied from the next update on: "none", "renormalize_l2_per_layer",
        "renormalize_l2_per_param_type", "clip_l2_per_layer" or "clip_l2_per_param_type" (the clip modes need a finite threshold > 0; the
        renormalize modes ignore it).  ClipElementWiseAbsoluteValue is `grad_clip` at construction, and excludes the L2 modes."""
        if mode not in GRADIENT_NORMALIZATIONS:
            raise ValueError(f"unknown gradient normalization {mode!r}; one of {sorted(GRADIENT_NORMALIZATIONS)} (element-wise clipping is grad_clip)")
        check(self.lib.b2g_net_set_gradient_normalization(self.h, GRADIENT_NORMALIZATIONS[mode], float(threshold)))

    def set_grad_allreduce(self, enabled: bool):
        """False = the reference's parameter-averaging mode: fit() updates locally, average_parameters() synchronises."""
        check(self.lib.b2g_net_set_grad_allreduce(self.h, int(enabled)))

    def set_sync_bn(self, enabled: bool):
        """Cross-replica BatchNorm statistics (SURVEY.md 8e): W ranks x N/W then equals 1 rank x N."""
        check(self.lib.b2g_net_set_sync_bn(self.h, int(enabled)))

    def set_grad_payload_bf16(self, enabled: bool):
        check(self.lib.b2g_net_set_grad_payload_bf16(self.h, int(enabled)))

    def enable_p2p_allreduce(self) -> bool:
        """COLLECTIVE (every rank, nets in the same order): gradient all-reduce as one kernel over NVLink peer memory (CUDA IPC) instead of
        ncclAllReduce; returns whether every rank could map its peers (otherwise all ranks stay on NCCL)."""
        out = C.c_int32(0)
        check(self.lib.b2g_net_enable_p2p_allreduce(self.h, C.byref(out)))
        return bool(out.value)

    def average_parameters(self):
        """ParameterAveragingTrainingMaster: params and updater state <- mean over ranks (J:325-330)."""
        check(self.lib.b2g_net_average_parameters(self.h))

    def iteration(self) -> int:
        """The updater's iteration counter (Adam's t - 1); part of a checkpoint."""
        v = C.c_int64()
        check(self.lib.b2g_net_get_iteration(self.h, C.byref(v)))
        return v.value

    def set_iteration(self, it: int):
        check(self.lib.b2g_net_set_iteration(self.h, int(it)))

    def dropout_pass(self) -> int:
        """The dropout pass counter P: train-mode forwards that applied a DropoutLayer mask; part of a checkpoint."""
        v = C.c_int64()
        check(self.lib.b2g_net_get_dropout_pass(self.h, C.byref(v)))
        return v.value

    def set_dropout_pass(self, p: int):
        check(self.lib.b2g_net_set_dropout_pass(self.h, int(p)))

    def simt_gemm_calls(self) -> int:
        """BF16 nets: GEMM-shaped operations that ran on the SIMT kernels instead of the tensor-core kernels since creation."""
        v = C.c_uint64()
        check(self.lib.b2g_net_simt_gemm_calls(self.h, C.byref(v)))
        return v.value

    def time_hbm_kernels(self, rows: int, channels: int, iters: int = 10):
        """(updater, BatchNorm apply, BatchNorm backward apply) ms per launch, each after an L2 flush.  Perturbs the parameters: bench only."""
        ms = np.zeros(3, np.float32)
        check(self.lib.b2g_test_hbm_kernels(self.h, rows, channels, iters, _fp(ms)))
        return [float(v) for v in ms]

    def weight_operand(self, layer: int, which: int, size: int) -> np.ndarray:
        """BF16 nets: the bf16 copy of layer `layer`'s W that the next forward reads (which = 0, internal [A][taps][B] order, `size` = W's
        element count), or the packed pixel-shuffle operand [(py,px,c)][(dyr,dxc)][O] of the <= 4-channel transposed conv (which = 1,
        `size` = 144 * O), widened to fp32."""
        out = np.empty(size, np.float32)
        check(self.lib.b2g_test_net_shadow(self.h, layer, which, _fp(out), out.size))
        return out

    def input_gradient(self, batch: int) -> np.ndarray:
        out = np.empty((batch, int(np.prod(self.input_shape))), np.float32)
        check(self.lib.b2g_net_get_input_gradient(self.h, batch, _fp(out)))
        return out

    def close(self):
        if self.h:
            self.lib.b2g_net_destroy(self.h)
            self.h = None


class Gan:
    """b2g_gan: the adversarial iteration J:408-471 with dis/gan/gen sharing storage."""

    def __init__(self, gen: Net, dis: Net, fake_bn_train: bool = False, use_cuda_graph: bool = True):
        self.gen, self.dis, self.lib = gen, dis, gen.lib
        cfg = GanConfig(int(fake_bn_train), int(use_cuda_graph))
        h = C.c_void_p()
        check(self.lib.b2g_gan_create(gen.h, dis.h, C.byref(cfg), C.byref(h)))
        self.h = h

    def step(self, x_real, z_d, z_g, y_real, y_fake, y_gen):
        a = [_f32(v) for v in (x_real, z_d, z_g, y_real, y_fake, y_gen)]
        losses = np.zeros(3, np.float32)
        check(self.lib.b2g_gan_step(self.h, *[_fp(v) for v in a], a[0].shape[0], _fp(losses)))
        return losses

    def step_ptr(self, ptrs, batch: int, losses: np.ndarray):
        """Raw-pointer variant for pinned host buffers (bench e2e): ptrs = 6 integer addresses."""
        args = [C.cast(C.c_void_p(p), C.POINTER(C.c_float)) for p in ptrs]
        check(self.lib.b2g_gan_step(self.h, *args, batch, _fp(losses)))

    def upload(self, x_real, z_d, z_g, y_real, y_fake, y_gen):
        a = [_f32(v) for v in (x_real, z_d, z_g, y_real, y_fake, y_gen)]
        check(self.lib.b2g_gan_upload(self.h, *[_fp(v) for v in a], a[0].shape[0]))
        self.gen.ctx.sync()

    def step_resident(self, batch: int):
        check(self.lib.b2g_gan_step_resident(self.h, batch))

    def losses(self) -> np.ndarray:
        out = np.zeros(3, np.float32)
        check(self.lib.b2g_gan_read_losses(self.h, _fp(out)))
        return out

    def last_step_ms(self) -> float:
        v = C.c_float()
        check(self.lib.b2g_gan_last_step_ms(self.h, C.byref(v)))
        return v.value

    def close(self):
        if self.h:
            self.lib.b2g_gan_destroy(self.h)
            self.h = None


def test_conv(ctx: Context, kind: int, impl: int, precision: int, geom: Dict[str, int], a, b, out_size: int, iters: int = 1):
    """Kernel-level hook: kind 0 fprop / 1 dgrad / 2 wgrad; impl 0 SIMT / 1 tensor-core. Returns (out, ms_per_iter)."""
    g = _lib.ConvGeom(**geom)
    a, b = _f32(a).ravel(), _f32(b).ravel()
    out = np.empty(out_size, np.float32)
    ms = C.c_float()
    check(ctx.lib.b2g_test_conv(ctx.h, kind, impl, precision, C.byref(g), _fp(a), _fp(b), _fp(out), iters, C.byref(ms)))
    return out, ms.value


EPI_PLAIN, EPI_STATS, EPI_BNBWD, EPI_ACTBWD = 0, 1, 2, 3


def test_conv_ex(ctx: Context, kind: int, geom: Dict[str, int], a, b, out_size: int, *, epi: int = 0, act: str = "identity", alpha: float = 0.0,
                 bias=None, scale=None, groups: int = 1, aux=None, aux2=None, iters: int = 1, impl: int = 1, bn: int = 0, max_ctas: int = 0,
                 poison: bool = False, w_mn: bool = False):
    """Tensor-core fprop (kind 0) / dgrad (kind 1) with the epilogue the training step uses (impl 3, kind 1: the pixel-shuffle deconv, b = the
    [O][4][4][C] weight).  bn forces the 64- / 128-column tile, max_ctas caps the persistent grid (0: production choice for both); poison
    fills the output with bf16 NaN before every launch; w_mn (kind 0, 1x1): b is the [C][O] dense weight.
    Returns (out, stats or None, kernel name, ms)."""
    g = _lib.ConvGeom(**geom)
    a, b = _f32(a).ravel(), _f32(b).ravel()
    out = np.empty(out_size, np.float32)
    oc = geom["o"] if kind == 0 else geom["c"]
    o = _lib.TestConvOpts()
    o.epi, o.act, o.alpha, o.groups = epi, ACTS[act], alpha, groups
    o.bn, o.max_ctas, o.poison, o.w_mn = bn, max_ctas, int(poison), int(w_mn)
    keep = []
    for name, v in (("bias", bias), ("scale", scale), ("aux", aux), ("aux2", aux2)):
        if v is not None:
            arr = _f32(v).ravel(); keep.append(arr); setattr(o, name, _fp(arr))
    stats = None
    if epi in (EPI_STATS, EPI_BNBWD):
        stats = np.zeros((groups, 2, oc), np.float64); o.stats = stats.ctypes.data_as(C.POINTER(C.c_double))
    ms = C.c_float()
    check(ctx.lib.b2g_test_conv_ex(ctx.h, kind, impl, BF16, C.byref(g), _fp(a), _fp(b), _fp(out), iters, C.byref(ms), C.byref(o)))
    return out, stats, o.kernel.decode(), ms.value


def test_bn(ctx: Context, precision: int, path: int, x, eps_out, gamma, beta, run_mean, run_var, *, act: str = "identity", alpha: float = 0.0,
            eps: float = 1e-5, decay: float = 0.9, g_gamma=None, g_beta=None, want_param_grads: bool = True):
    """One BatchNorm(+activation) forward and backward through the training-step kernels (b2g_test_bn).  x, eps_out: [groups, rows, C].
    Returns a dict with y, eps_in ([groups, rows, C]), g_gamma, g_beta (accumulated into the given initial values), g_mean, g_var ([C]) and
    mean, invstd ([groups, C])."""
    x, e = _f32(x), _f32(eps_out)
    groups, rows, ch = x.shape
    par = [_f32(v).ravel() for v in (gamma, beta, run_mean, run_var)]
    r = {k: np.empty(x.shape, np.float32) for k in ("y", "eps_in")}
    r["g_gamma"] = _f32(np.zeros(ch) if g_gamma is None else g_gamma).copy()
    r["g_beta"] = _f32(np.zeros(ch) if g_beta is None else g_beta).copy()
    r.update({k: np.empty(ch, np.float32) for k in ("g_mean", "g_var")})
    r.update({k: np.empty((groups, ch), np.float32) for k in ("mean", "invstd")})
    check(ctx.lib.b2g_test_bn(ctx.h, precision, path, groups, rows, ch, _fp(x), _fp(e), *[_fp(v) for v in par], ACTS[act], alpha, eps, decay,
                              int(want_param_grads), *[_fp(r[k]) for k in ("y", "eps_in", "g_gamma", "g_beta", "g_mean", "g_var", "mean", "invstd")]))
    return r


def test_dropout(ctx: Context, precision: int, x, dy, p: float, *, seed: int = 666, layer: int = 0, rank: int = 0, pass_: int = 0):
    """One DropoutLayer forward and backward through the training-step kernels (b2g_test_dropout).  x, dy: [rows, H, W, C] in the engine's NHWC
    order (or [rows, F]).  Returns (y, dx) in the same shape."""
    x, e = _f32(x), _f32(dy)
    rows = x.shape[0]
    h, w, c = (x.shape[1:] if x.ndim == 4 else (1, 1, int(np.prod(x.shape[1:]))))
    y, dx = np.empty_like(x), np.empty_like(x)
    check(ctx.lib.b2g_test_dropout(ctx.h, precision, seed, layer, rank, pass_, rows, h, w, c, p, _fp(x), _fp(e), _fp(y), _fp(dx)))
    return y, dx
