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


class ConvGeom(C.Structure):
    _fields_ = [(k, C.c_int32) for k in ("n", "h", "w", "c", "oh", "ow", "o", "kh", "kw", "sh", "sw", "ph", "pw")]


class TestConvOpts(C.Structure):
    """b2g_test_conv_opts: the epilogue a kernel-level parity test asks for, the name of the kernel that ran, and the schedule controls
    (forced tile width, grid cap, output poisoning, [C][O] dense weight operand)."""
    _fields_ = [("epi", C.c_int32), ("act", C.c_int32), ("alpha", C.c_float), ("bias", C.POINTER(C.c_float)), ("scale", C.POINTER(C.c_float)),
                ("groups", C.c_int32), ("aux", C.POINTER(C.c_float)), ("aux2", C.POINTER(C.c_float)), ("stats", C.POINTER(C.c_double)), ("kernel", C.c_char * 64),
                ("bn", C.c_int32), ("max_ctas", C.c_int32), ("poison", C.c_int32), ("w_mn", C.c_int32)]


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
    "b2g_net_get_updater_state": (_i32, [_vp, _fp, _i64]),
    "b2g_net_set_updater_state": (_i32, [_vp, _fp, _i64]),
    "b2g_net_output": (_i32, [_vp, _fp, _i32, _i32, _fp]),
    "b2g_net_get_activation": (_i32, [_vp, _i32, _i32, _fp]),
    "b2g_net_compute_gradient_and_score": (_i32, [_vp, _fp, _fp, _i32, _fp]),
    "b2g_net_get_input_gradient": (_i32, [_vp, _i32, _fp]),
    "b2g_net_fit": (_i32, [_vp, _fp, _fp, _i32, _fp]),
    "b2g_net_get_iteration": (_i32, [_vp, C.POINTER(_i64)]),
    "b2g_net_set_iteration": (_i32, [_vp, _i64]),
    "b2g_net_get_dropout_pass": (_i32, [_vp, C.POINTER(_i64)]),
    "b2g_net_set_dropout_pass": (_i32, [_vp, _i64]),
    "b2g_net_set_gradient_normalization": (_i32, [_vp, _i32, C.c_float]),
    "b2g_net_simt_gemm_calls": (_i32, [_vp, C.POINTER(C.c_uint64)]),
    "b2g_gan_create": (_i32, [_vp, _vp, C.POINTER(GanConfig), _pvp]),
    "b2g_gan_destroy": (_i32, [_vp]),
    "b2g_gan_step": (_i32, [_vp, _fp, _fp, _fp, _fp, _fp, _fp, _i32, _fp]),
    "b2g_gan_upload": (_i32, [_vp, _fp, _fp, _fp, _fp, _fp, _fp, _i32]),
    "b2g_gan_step_resident": (_i32, [_vp, _i32]),
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
    "b2g_test_net_shadow": (_i32, [_vp, _i32, _i32, _fp, _i64]),
    "b2g_test_dropout": (_i32, [_vp, _i32, C.c_uint64, _i32, _i32, _i64, _i32, _i32, _i32, _i32, C.c_float, _fp, _fp, _fp, _fp]),
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
