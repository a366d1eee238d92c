"""ctypes binding of include/mnn_b200.h -- the same C ABI the MNN plugin binds (see INTEGRATION.md).

The product path is CUDA only: importing this module builds nothing and falls back to nothing.  If
libmnn_b200.so is missing or no sm_90 device is present every entry point raises.
"""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("MNNB200_LIB") or os.path.join(HERE, "libmnn_b200.so")   # MNNB200_LIB: an A/B measurement build


class MnnB200Error(RuntimeError):
    pass


class ConvDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("ic", "oc", "kh", "kw", "stride_h", "stride_w", "pad_h", "pad_w",
                                         "dilate_h", "dilate_w", "group", "relu")]


_lib = None

# name -> (restype, argtypes); every symbol include/mnn_b200.h declares
P = C.c_void_p
_RESIZE = [P, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, C.c_float, C.c_int, C.c_int, C.c_int,
           C.POINTER(C.c_int), C.POINTER(C.c_int)]
SIGNATURES = {
    "mnnb200_last_error": (C.c_char_p, []),
    "mnnb200_abi_version": (C.c_int, []),
    "mnnb200_runtime_create": (C.c_int, [C.c_int, P, C.POINTER(P)]),
    "mnnb200_runtime_destroy": (None, [P]),
    "mnnb200_runtime_stream": (P, [P]),
    "mnnb200_runtime_sync": (C.c_int, [P]),
    "mnnb200_runtime_info": (C.c_int, [P, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int),
                                       C.POINTER(C.c_size_t)]),
    "mnnb200_alloc": (C.c_int, [P, C.c_size_t, C.POINTER(P)]),
    "mnnb200_free": (C.c_int, [P, P]),
    "mnnb200_memcpy_h2d": (C.c_int, [P, P, P, C.c_size_t]),
    "mnnb200_memcpy_d2h": (C.c_int, [P, P, P, C.c_size_t]),
    "mnnb200_nhwc16_bytes": (C.c_size_t, [C.c_int] * 4),
    "mnnb200_launch_count": (C.c_ulonglong, []),
    "mnnb200_graph_begin_capture": (C.c_int, [P]),
    "mnnb200_graph_end_capture": (C.c_int, [P, C.POINTER(P)]),
    "mnnb200_graph_launch": (C.c_int, [P, P]),
    "mnnb200_graph_destroy": (None, [P]),
    "mnnb200_host_register": (C.c_int, [P, P, C.c_size_t]),
    "mnnb200_host_unregister": (C.c_int, [P, P]),
    "mnnb200_alloc_host": (C.c_int, [P, C.c_size_t, C.POINTER(P)]),
    "mnnb200_free_host": (C.c_int, [P, P]),
    "mnnb200_runtime_mark_begin": (C.c_int, [P]),
    "mnnb200_runtime_mark_end": (C.c_int, [P]),
    "mnnb200_runtime_last_gpu_ms": (C.c_float, [P]),
    "mnnb200_float_to_int8": (C.c_int, [P, P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int,
                                        C.c_int, P]),
    "mnnb200_int8_to_float": (C.c_int, [P, P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, P]),
    "mnnb200_pack_nchw_int8": (C.c_int, [P, P, C.c_int, C.c_int, C.c_int, C.c_int, P]),
    "mnnb200_unpack_nchw_int8": (C.c_int, [P, P, C.c_int, C.c_int, C.c_int, C.c_int, P]),
    "mnnb200_conv_int8_create": (C.c_int, [P, C.POINTER(ConvDesc), P, P, P, C.POINTER(P)]),
    "mnnb200_conv_int8_create_legacy": (C.c_int, [P, C.POINTER(ConvDesc), P, P, P, C.POINTER(P)]),
    "mnnb200_conv_int8_resize": (C.c_int, _RESIZE),
    "mnnb200_conv_int8_execute": (C.c_int, [P, P, P]),
    "mnnb200_conv_int8_set_pad": (C.c_int, [P, C.c_int, C.c_int]),
    "mnnb200_conv_int8_set_variant": (C.c_int, [P, C.c_int]),
    "mnnb200_conv_group_create": (C.c_int, [P, C.POINTER(P), C.c_int, C.POINTER(P)]),
    "mnnb200_conv_group_bind": (C.c_int, [P, C.POINTER(P), C.POINTER(P)]),
    "mnnb200_conv_group_execute": (C.c_int, [P]),
    "mnnb200_conv_int8_groupable": (C.c_int, [P]),
    "mnnb200_conv_int8_group_plan": (C.c_int, [P, C.POINTER(C.c_int), C.c_int]),
    "mnnb200_conv_int8_wino_create": (C.c_int, [P, C.POINTER(ConvDesc), P, P, P, P, C.c_int, C.POINTER(P)]),
    "mnnb200_conv_int8_wino_resize": (C.c_int, _RESIZE),
    "mnnb200_conv_int8_wino_execute": (C.c_int, [P, P, P]),
    "mnnb200_conv_int8_wino_execute_phases": (C.c_int, [P, P, P, C.c_int]),
    "mnnb200_conv_int8_wino_plan": (C.c_int, [P, C.POINTER(C.c_int), C.c_int]),
    "mnnb200_exec_cost": (C.c_int, [P, C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "mnnb200_dwconv_int8_create": (C.c_int, [P, C.POINTER(ConvDesc), P, P, P, C.POINTER(P)]),
    "mnnb200_dwconv_int8_resize": (C.c_int, _RESIZE),
    "mnnb200_dwconv_int8_execute": (C.c_int, [P, P, P]),
    "mnnb200_binary_add_int8": (C.c_int, [P, P, C.c_float, C.c_int, P, C.c_float, C.c_int, P, C.c_float, C.c_int, C.c_int,
                                          C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "mnnb200_avgpool_int8": (C.c_int, [P, P] + [C.c_int] * 12 + [C.c_float] * 4 + [C.c_int, C.c_int, P, C.c_int, C.c_int]),
    "mnnb200_softmax_int8": (C.c_int, [P, P, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int, C.c_int, P]),
    "mnnb200_scale_int8_create": (C.c_int, [P, C.c_int, P, P, C.POINTER(P)]),
    "mnnb200_scale_int8_resize": (C.c_int, [P, C.c_float, C.c_int, C.c_float, C.c_int, C.c_int, C.c_int]),
    "mnnb200_scale_int8_execute": (C.c_int, [P, P, C.c_int, C.c_int, C.c_int, P]),
    "mnnb200_pool_int8": (C.c_int, [P, P] + [C.c_int] * 11 + [P, C.c_int, C.c_int]),
    "mnnb200_relu_f32": (C.c_int, [P, P, C.c_size_t, C.c_float, P]),
    "mnnb200_reduce_f32": (C.c_int, [P, P, C.c_int, C.c_int, C.c_int, C.c_int, P]),
    "mnnb200_pool_f32": (C.c_int, [P, P] + [C.c_int] * 13 + [P, C.c_int, C.c_int]),
    "mnnb200_raster_b32": (C.c_int, [P, P, C.c_int, P, C.c_size_t, C.c_int]),
    "mnnb200_transpose_b32": (C.c_int, [P, P, C.c_int, C.c_int, C.c_int, P]),
    "mnnb200_memcpy_d2d": (C.c_int, [P, P, P, C.c_size_t]),
    "mnnb200_linear_w8_create": (C.c_int, [P, C.c_int, C.c_int, P, P, P, P, C.c_int, C.c_int, C.POINTER(P)]),
    "mnnb200_linear_w8_create_blocked": (C.c_int, [P, C.c_int, C.c_int, C.c_int, P, P, P, P, C.c_int, C.c_int, C.POINTER(P)]),
    "mnnb200_linear_w8_resize": (C.c_int, [P, C.c_int]),
    "mnnb200_linear_w8_execute": (C.c_int, [P, P, P]),
    "mnnb200_matmul_create": (C.c_int, [P] + [C.c_int] * 7 + [C.POINTER(P)]),
    "mnnb200_matmul_execute": (C.c_int, [P, P, P, P, P]),
    "mnnb200_conv_f32_create": (C.c_int, [P, C.POINTER(ConvDesc), P, P, C.c_int, C.POINTER(P)]),
    "mnnb200_conv_f32_set_pad": (C.c_int, [P, C.c_int, C.c_int]),
    "mnnb200_conv_f32_resize": (C.c_int, [P, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "mnnb200_conv_f32_execute": (C.c_int, [P, P, P]),
    "mnnb200_conv_f32_plan": (C.c_int, [P, C.POINTER(C.c_int), C.c_int]),
    "mnnb200_dwconv_f32_create": (C.c_int, [P, C.POINTER(ConvDesc), P, P, C.c_int, C.POINTER(P)]),
    "mnnb200_dwconv_f32_resize": (C.c_int, [P, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "mnnb200_dwconv_f32_execute": (C.c_int, [P, P, P]),
    "mnnb200_binary_add_f32": (C.c_int, [P, P, P, P, C.c_size_t]),
    "mnnb200_scale_f32_create": (C.c_int, [P, C.c_int, P, P, C.POINTER(P)]),
    "mnnb200_scale_f32_resize": (C.c_int, [P, C.c_int, C.c_int, C.c_int]),
    "mnnb200_scale_f32_execute": (C.c_int, [P, P, P]),
    "mnnb200_softmax_f32": (C.c_int, [P, P, C.c_int, C.c_int, C.c_int, P]),
    "mnnb200_binary_f32": (C.c_int, [P, C.c_int, P, C.c_size_t, P, C.c_size_t, P, C.c_size_t, C.c_int]),
    "mnnb200_unary_f32": (C.c_int, [P, C.c_int, P, P, C.c_size_t]),
    "mnnb200_argmax_f32": (C.c_int, [P, P, C.c_int, C.c_int, C.c_int, C.c_int, P]),
    "mnnb200_exec_destroy": (None, [P]),
}


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise MnnB200Error(f"{LIB_PATH} is missing: run `python -m mnn_b200.build` (there is no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)  # AttributeError if the library does not export a declared symbol
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(status, what=""):
    if status != 0:
        msg = lib().mnnb200_last_error().decode(errors="replace")
        raise MnnB200Error(f"{what} failed with status {status}: {msg}")
