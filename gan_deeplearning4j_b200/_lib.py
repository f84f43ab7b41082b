"""ctypes binding of libb200gan.so -- the same C-ABI (include/b200gan.h) the JNI shim exposes to the Java facade.

There is no CPU fallback: importing works anywhere (so that symbol/ABI tests run without a GPU), but every
compute entry point needs the CUDA library and an sm_90 device and raises B200GanError otherwise.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libb200gan.so")
NAME_LEN = 64


class B200GanError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"libb200gan error {code}: {msg}")
        self.code = code


class LayerDesc(C.Structure):
    _fields_ = [("type", C.c_int32), ("name", C.c_char * NAME_LEN), ("n_in", C.c_int32), ("n_out", C.c_int32),
                ("k_h", C.c_int32), ("k_w", C.c_int32), ("s_h", C.c_int32), ("s_w", C.c_int32), ("p_h", C.c_int32), ("p_w", C.c_int32),
                ("has_bias", C.c_int32), ("act", C.c_int32), ("act_alpha", C.c_float), ("updater", C.c_int32),
                ("lr", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float), ("l2", C.c_float),
                ("bn_decay", C.c_float), ("bn_eps", C.c_float), ("pre_h", C.c_int32), ("pre_w", C.c_int32), ("pre_c", C.c_int32),
                ("loss", C.c_int32), ("frozen", C.c_int32)]


class NetConfig(C.Structure):
    _fields_ = [("in_h", C.c_int32), ("in_w", C.c_int32), ("in_c", C.c_int32), ("max_batch", C.c_int32), ("precision", C.c_int32),
                ("grad_clip", C.c_float), ("xent_clip_eps", C.c_float), ("bn_groups", C.c_int32), ("seed", C.c_uint64)]


class GanConfig(C.Structure):
    _fields_ = [("fake_bn_train", C.c_int32), ("use_cuda_graph", C.c_int32)]


class LrSchedule(C.Structure):
    """b2g_lr_schedule: one DL4J ISchedule (kind, ScheduleType, its parameters, and a MapSchedule's entries, copied during the call)."""
    _fields_ = [("kind", C.c_int32), ("type", C.c_int32), ("initial", C.c_double), ("gamma", C.c_double), ("power", C.c_double),
                ("step", C.c_double), ("decay_rate", C.c_double), ("n_map", C.c_int32), ("map_keys", C.POINTER(C.c_int32)),
                ("map_values", C.POINTER(C.c_double))]


class WeightNoise(C.Structure):
    """b2g_weight_noise: DropConnect (p, or an ISchedule copied during the call) or WeightNoise (a distribution's two parameters)."""
    _fields_ = [("kind", C.c_int32), ("apply_to_bias", C.c_int32), ("p", C.c_float), ("p_schedule", C.POINTER(LrSchedule)), ("dist", C.c_int32),
                ("a", C.c_float), ("b", C.c_float), ("additive", C.c_int32)]


class WeightInit(C.Structure):
    """b2g_weight_init: a WeightInit scheme, DISTRIBUTION's distribution and its two parameters, and biasInit."""
    _fields_ = [("scheme", C.c_int32), ("dist", C.c_int32), ("a", C.c_float), ("b", C.c_float), ("bias_init", C.c_float)]


class Regularization(C.Structure):
    """b2g_regularization: l1 and l2 on W, l1_bias and l2_bias on b."""
    _fields_ = [("l1", C.c_float), ("l2", C.c_float), ("l1_bias", C.c_float), ("l2_bias", C.c_float)]


class Constraint(C.Structure):
    """b2g_constraint: one DL4J LayerConstraint on one parameter tensor (kind, DL4J dimensions as a bit mask, bounds, MinMaxNorm's rate)."""
    _fields_ = [("kind", C.c_int32), ("dims_mask", C.c_int32), ("max_norm", C.c_double), ("min_norm", C.c_double), ("rate", C.c_double)]


class ConvGeom(C.Structure):
    _fields_ = [(k, C.c_int32) for k in ("n", "h", "w", "c", "oh", "ow", "o", "kh", "kw", "sh", "sw", "ph", "pw")]


class TestConvOpts(C.Structure):
    """b2g_test_conv_opts: the epilogue a kernel-level parity test asks for, the name of the kernel that ran, and the schedule controls
    (forced tile width, grid cap, output poisoning, [C][O] dense weight operand); the parameter offset of the SIMT / skinny-layer / dense
    kernels' fp32 weight operand or gradient, and the split-K count they report."""
    _fields_ = [("epi", C.c_int32), ("act", C.c_int32), ("alpha", C.c_float), ("bias", C.POINTER(C.c_float)), ("scale", C.POINTER(C.c_float)),
                ("groups", C.c_int32), ("aux", C.POINTER(C.c_float)), ("aux2", C.POINTER(C.c_float)), ("stats", C.POINTER(C.c_double)), ("kernel", C.c_char * 64),
                ("bn", C.c_int32), ("max_ctas", C.c_int32), ("poison", C.c_int32), ("w_mn", C.c_int32), ("per_tap", C.c_int32), ("slab", C.c_int32),
                ("defer", C.c_int32), ("db", C.POINTER(C.c_float)), ("param_offset", C.c_int32), ("splits", C.c_int32)]


class EwReduceJob(C.Structure):
    """b2g_ew_reduce_job: one split-K sum of a reduce list (offsets into one buffer); `wide` is set by the call."""
    _fields_ = [("n", C.c_int64), ("stride", C.c_int64), ("src_off", C.c_int64), ("dst_off", C.c_int64), ("splits", C.c_int32), ("wide", C.c_int32)]


class TestEwOpts(C.Structure):
    """b2g_test_ew_opts: which reduction / loss / element-wise kernel wrapper to run, its sizes and options, and what ran."""
    _fields_ = [("op", C.c_int32), ("n", C.c_int64), ("rows", C.c_int32), ("cols", C.c_int32), ("groups", C.c_int32), ("splits", C.c_int32),
                ("stride", C.c_int64)] + [(k, C.c_int32) for k in ("N", "H", "W", "C", "KH", "KW", "SH", "SW", "act")] + [
                ("alpha", C.c_float), ("clip_eps", C.c_float), ("offset", C.c_int32), ("in_place", C.c_int32), ("accumulate", C.c_int32),
                ("poison", C.c_int32), ("n_jobs", C.c_int32), ("jobs", C.POINTER(EwReduceJob)), ("n_seg", C.c_int32),
                ("seg_off", C.POINTER(C.c_int64)), ("seg_len", C.POINTER(C.c_int64)), ("seg_coef", C.POINTER(C.c_float)), ("sumsq", C.c_double),
                ("kernel", C.c_char * 64), ("loss", C.c_int32)]


class TestPoolOpts(C.Structure):
    """b2g_test_pool_opts: which pooling kernels to run (pool2d / global), the kind, p, geometry and switches, and what ran."""
    _fields_ = [("op", C.c_int32), ("pool", C.c_int32), ("pnorm", C.c_float)] + [
                (k, C.c_int32) for k in ("N", "H", "W", "C", "KH", "KW", "SH", "SW", "PH", "PW", "offset", "poison")] + [
                ("kernel", C.c_char * 64), ("splits", C.c_int32)]


class TestBnOpts(C.Structure):
    """b2g_test_bn_opts: the accumulator path, replica count, per-replica shape, fused activation and BatchNorm constants of a cross-replica
    BatchNorm test."""
    _fields_ = [(k, C.c_int32) for k in ("path", "replicas", "groups", "rows", "C", "act")] + [
                ("alpha", C.c_float), ("eps", C.c_float), ("decay", C.c_float), ("want_param_grads", C.c_int32)]


class TestLossOpts(C.Structure):
    """b2g_test_loss_opts: which weighted / masked loss kernel to run, its sizes and options, and what ran."""
    _fields_ = [(k, C.c_int32) for k in ("kernel", "rows", "cols", "groups", "loss", "act")] + [("alpha", C.c_float), ("clip_eps", C.c_float)] + [
                (k, C.c_int32) for k in ("mask_width", "offset", "poison")] + [("kernel_name", C.c_char * 64)]


_vp, _i32, _i64, _fp = C.c_void_p, C.c_int32, C.c_int64, C.POINTER(C.c_float)
_pvp = C.POINTER(C.c_void_p)

# name -> (restype, argtypes); every symbol include/b200gan.h declares
PROTOTYPES = {
    "b2g_version": (_i32, []),
    "b2g_ctx_create": (_i32, [_i32, _pvp]),
    "b2g_ctx_destroy": (_i32, [_vp]),
    "b2g_last_error": (C.c_char_p, []),
    "b2g_sync": (_i32, [_vp]),
    "b2g_launch_count": (_i32, [_vp, C.POINTER(C.c_uint64)]),
    "b2g_timer_start": (_i32, [_vp]),
    "b2g_timer_stop_ms": (_i32, [_vp, _fp]),
    "b2g_flush_l2": (_i32, [_vp]),
    "b2g_device_info": (_i32, [_vp, C.POINTER(_i32), C.POINTER(_i32), C.POINTER(_i32), C.POINTER(C.c_uint64)]),
    "b2g_net_create": (_i32, [_vp, C.POINTER(NetConfig), C.POINTER(LayerDesc), _i32, _pvp]),
    "b2g_net_destroy": (_i32, [_vp]),
    "b2g_net_num_params": (_i32, [_vp, C.POINTER(_i64)]),
    "b2g_net_output_size": (_i32, [_vp, C.POINTER(_i64)]),
    "b2g_net_layer_output_size": (_i32, [_vp, _i32, C.POINTER(_i64)]),
    "b2g_net_set_param": (_i32, [_vp, C.c_char_p, C.c_char_p, _fp, _i64]),
    "b2g_net_get_param": (_i32, [_vp, C.c_char_p, C.c_char_p, _fp, _i64]),
    "b2g_net_get_params": (_i32, [_vp, _fp, _i64]),
    "b2g_net_set_params": (_i32, [_vp, _fp, _i64]),
    "b2g_net_get_gradients": (_i32, [_vp, _fp, _i64]),
    "b2g_net_updater_state_size": (_i32, [_vp, C.POINTER(_i64)]),
    "b2g_net_get_updater_state": (_i32, [_vp, _fp, _i64]),
    "b2g_net_set_updater_state": (_i32, [_vp, _fp, _i64]),
    "b2g_net_output": (_i32, [_vp, _fp, _i32, _i32, _fp]),
    "b2g_net_get_activation": (_i32, [_vp, _i32, _i32, _fp]),
    "b2g_net_compute_gradient_and_score": (_i32, [_vp, _fp, _fp, _i32, _fp]),
    "b2g_net_get_input_gradient": (_i32, [_vp, _i32, _fp]),
    "b2g_net_fit": (_i32, [_vp, _fp, _fp, _i32, _fp]),
    "b2g_net_fit_masked": (_i32, [_vp, _fp, _fp, _i32, _fp, _fp, _i32]),
    "b2g_net_compute_gradient_and_score_masked": (_i32, [_vp, _fp, _fp, _i32, _fp, _fp, _i32]),
    "b2g_net_set_loss_weights": (_i32, [_vp, C.c_char_p, _fp, _i32]),
    "b2g_net_loss_columns": (_i32, [_vp, C.POINTER(C.c_int32)]),
    "b2g_net_get_iteration": (_i32, [_vp, C.POINTER(_i64)]),
    "b2g_net_set_iteration": (_i32, [_vp, _i64]),
    "b2g_net_get_dropout_pass": (_i32, [_vp, C.POINTER(_i64)]),
    "b2g_net_set_dropout_pass": (_i32, [_vp, _i64]),
    "b2g_net_set_gradient_normalization": (_i32, [_vp, _i32, C.c_float]),
    "b2g_net_set_lr_schedule": (_i32, [_vp, C.c_char_p, C.POINTER(LrSchedule)]),
    "b2g_net_set_constraints": (_i32, [_vp, C.c_char_p, C.c_char_p, C.POINTER(Constraint), _i32]),
    "b2g_net_apply_constraints": (_i32, [_vp]),
    "b2g_net_get_learning_rate": (_i32, [_vp, C.c_char_p, _fp]),
    "b2g_net_set_dropout_schedule": (_i32, [_vp, C.c_char_p, C.POINTER(LrSchedule)]),
    "b2g_net_get_dropout_value": (_i32, [_vp, C.c_char_p, _fp]),
    "b2g_net_set_weight_noise": (_i32, [_vp, C.c_char_p, C.POINTER(WeightNoise)]),
    "b2g_net_init_weights": (_i32, [_vp, C.c_char_p, C.POINTER(WeightInit)]),
    "b2g_net_set_regularization": (_i32, [_vp, C.c_char_p, C.POINTER(Regularization)]),
    "b2g_net_get_regularization": (_i32, [_vp, C.c_char_p, C.POINTER(Regularization)]),
    "b2g_net_calc_regularization": (_i32, [_vp, C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "b2g_net_get_epoch": (_i32, [_vp, C.POINTER(_i64)]),
    "b2g_net_set_epoch": (_i32, [_vp, _i64]),
    "b2g_net_simt_gemm_calls": (_i32, [_vp, C.POINTER(C.c_uint64)]),
    "b2g_gan_create": (_i32, [_vp, _vp, C.POINTER(GanConfig), _pvp]),
    "b2g_gan_destroy": (_i32, [_vp]),
    "b2g_gan_step": (_i32, [_vp, _fp, _fp, _fp, _fp, _fp, _fp, _i32, _fp]),
    "b2g_gan_upload": (_i32, [_vp, _fp, _fp, _fp, _fp, _fp, _fp, _i32]),
    "b2g_gan_step_resident": (_i32, [_vp, _i32]),
    "b2g_gan_set_label_masks": (_i32, [_vp, _fp, _fp, _fp, _i32, _i32]),
    "b2g_gan_read_losses": (_i32, [_vp, _fp]),
    "b2g_gan_last_step_ms": (_i32, [_vp, _fp]),
    "b2g_comm_unique_id": (_i32, [_vp]),
    "b2g_ctx_comm_init": (_i32, [_vp, _i32, _i32, _vp]),
    "b2g_ctx_comm_destroy": (_i32, [_vp]),
    "b2g_net_set_grad_allreduce": (_i32, [_vp, _i32]),
    "b2g_net_average_parameters": (_i32, [_vp]),
    "b2g_net_set_sync_bn": (_i32, [_vp, _i32]),
    "b2g_net_set_grad_payload_bf16": (_i32, [_vp, _i32]),
    "b2g_net_enable_p2p_allreduce": (_i32, [_vp, C.POINTER(C.c_int32)]),
    "b2g_ctx_allreduce_test": (_i32, [_vp, _fp, _i64]),
    "b2g_test_conv": (_i32, [_vp, _i32, _i32, _i32, C.POINTER(ConvGeom), _fp, _fp, _fp, _i32, _fp]),
    "b2g_test_hbm_kernels": (_i32, [_vp, _i32, _i32, _i32, _fp]),
    "b2g_test_conv_ex": (_i32, [_vp, _i32, _i32, _i32, C.POINTER(ConvGeom), _fp, _fp, _fp, _i32, _fp, C.POINTER(TestConvOpts)]),
    "b2g_test_bn": (_i32, [_vp, _i32, _i32, _i32, _i32, _i32, _fp, _fp, _fp, _fp, _fp, _fp, _i32, C.c_float, C.c_float, C.c_float,
                           _i32, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp]),
    "b2g_test_bn_ex": (_i32, [_vp, C.POINTER(TestBnOpts)] + [_fp] * 16),
    "b2g_test_net_shadow": (_i32, [_vp, _i32, _i32, _fp, _i64]),
    "b2g_test_net_noisy_operand": (_i32, [_vp, _i32, _i32, _fp, _i64]),
    "b2g_test_dropout": (_i32, [_vp, _i32, C.c_uint64, _i32, _i32, _i64, _i32, _i32, _i32, _i32, C.c_float, _fp, _fp, _fp, _fp]),
    "b2g_test_dropout_kind": (_i32, [_vp, _i32, _i32, C.c_uint64, _i32, _i32, _i64, _i32, _i32, _i32, _i32, C.c_float, _fp, _fp, _fp, _fp]),
    "b2g_test_ew": (_i32, [_vp, _i32, C.POINTER(TestEwOpts), _fp, _fp, _fp, _fp, _fp]),
    "b2g_test_pool": (_i32, [_vp, _i32, C.POINTER(TestPoolOpts), _fp, _fp, _fp, _fp, _fp]),
    "b2g_test_loss": (_i32, [_vp, _i32, C.POINTER(TestLossOpts), _fp, _fp, _fp, _fp, _fp, _fp]),
}

_lib = None


def load():
    """Load libb200gan.so (built in-tree by `make` / __graft_entry__.build()). Fails loudly if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise B200GanError(-7, f"{LIB_PATH} is missing: build it with `make` (nvcc, sm_90a). There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)        # AttributeError if the library does not export a declared symbol
        fn.restype, fn.argtypes = res, args
    _lib = lib
    return lib


def check(code):
    if code != 0:
        raise B200GanError(code, load().b2g_last_error().decode(errors="replace"))
