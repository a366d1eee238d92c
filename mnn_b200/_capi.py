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


class RopeNorm(C.Structure):
    _fields_ = [("gamma", C.c_void_p), ("beta", C.c_void_p), ("size", C.c_int32), ("eps", C.c_float), ("rms", C.c_int32)]


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
    "mnnb200_conv_group_schedule": (C.c_int, [C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int, C.c_int, C.POINTER(C.c_uint32), C.c_int,
                                              C.POINTER(C.c_int), C.POINTER(C.c_int)]),
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
    "mnnb200_linear_w4_create_blocked": (C.c_int, [P, C.c_int, C.c_int, C.c_int, P, P, P, P, C.c_int, C.c_int, C.POINTER(P)]),
    "mnnb200_linear_w8_resize": (C.c_int, [P, C.c_int]),
    "mnnb200_linear_w8_execute": (C.c_int, [P, P, P]),
    "mnnb200_linear_w8_plan": (C.c_int, [P, C.POINTER(C.c_int), C.c_int]),
    "mnnb200_matmul_create": (C.c_int, [P] + [C.c_int] * 7 + [C.POINTER(P)]),
    "mnnb200_matmul_execute": (C.c_int, [P, P, P, P, P]),
    "mnnb200_matmul_create_broadcast": (C.c_int, [P, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)] +
                                        [C.c_int] * 5 + [C.POINTER(P)]),
    "mnnb200_conv_f32_create": (C.c_int, [P, C.POINTER(ConvDesc), P, P, C.c_int, C.POINTER(P)]),
    "mnnb200_conv_f32_create_grouped": (C.c_int, [P, C.POINTER(ConvDesc), P, P, C.c_int, C.POINTER(P)]),
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


# libmnn_b200_deconv.so (include/mnn_b200_deconv.h): the float Deconvolution executions, on the runtime and execution handles above
DECONV_LIB_PATH = os.path.join(os.path.dirname(LIB_PATH), "libmnn_b200_deconv.so")
DECONV_SIGNATURES = {
    "mnnb200_deconv_f32_create": (C.c_int, [P, C.POINTER(ConvDesc), P, P, C.c_int, C.POINTER(P)]),
    "mnnb200_deconv_f32_set_pad": (C.c_int, [P, C.c_int, C.c_int]),
    "mnnb200_deconv_f32_resize": (C.c_int, [P, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "mnnb200_deconv_f32_execute": (C.c_int, [P, P, P]),
    "mnnb200_deconv_f32_plan": (C.c_int, [P, C.POINTER(C.c_int), C.c_int]),
    "mnnb200_dwdeconv_f32_create": (C.c_int, [P, C.POINTER(ConvDesc), P, P, C.c_int, C.POINTER(P)]),
    "mnnb200_dwdeconv_f32_resize": (C.c_int, [P, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "mnnb200_dwdeconv_f32_execute": (C.c_int, [P, P, P]),
}
_deconv_lib = None

# libmnn_b200_interp.so (include/mnn_b200_interp.h): the float Interp execution, on the runtime and execution handles above
INTERP_LIB_PATH = os.path.join(os.path.dirname(LIB_PATH), "libmnn_b200_interp.so")
INTERP_SIGNATURES = {
    "mnnb200_interp_f32_create": (C.c_int, [P, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, C.POINTER(P)]),
    "mnnb200_interp_f32_resize": (C.c_int, [P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "mnnb200_interp_f32_execute": (C.c_int, [P, P, P]),
    "mnnb200_interp_f32_plan": (C.c_int, [P, C.POINTER(C.c_int), C.c_int]),
}
_interp_lib = None

# libmnn_b200_gather.so (include/mnn_b200_gather.h): the gathers and the int32 / fp32 Cast, on the runtime and execution handles above
GATHER_LIB_PATH = os.path.join(os.path.dirname(LIB_PATH), "libmnn_b200_gather.so")
GATHER_SIGNATURES = {
    "mnnb200_gather_create": (C.c_int, [P, C.c_int, C.POINTER(P)]),
    "mnnb200_gather_resize": (C.c_int, [P, C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int), C.c_int, C.c_int]),
    "mnnb200_gather_execute": (C.c_int, [P, P, P, P]),
    "mnnb200_gather_plan": (C.c_int, [P, C.POINTER(C.c_int), C.c_int]),
    "mnnb200_cast_i32_f32": (C.c_int, [P, P, P, C.c_longlong]),
    "mnnb200_cast_f32_i32": (C.c_int, [P, P, P, C.c_longlong]),
}
_gather_lib = None

# libmnn_b200_scatter.so (include/mnn_b200_scatter.h): ScatterNd and ScatterElements, on the runtime and execution handles above
SCATTER_LIB_PATH = os.path.join(os.path.dirname(LIB_PATH), "libmnn_b200_scatter.so")
_IP = C.POINTER(C.c_int)
SCATTER_SIGNATURES = {
    "mnnb200_scatter_create": (C.c_int, [P, C.c_int, C.c_int, C.c_int, C.POINTER(P)]),
    "mnnb200_scatter_resize": (C.c_int, [P, _IP, C.c_int, _IP, C.c_int, _IP, C.c_int, C.c_int, C.c_int]),
    "mnnb200_scatter_execute": (C.c_int, [P, P, P, P, P]),
    "mnnb200_scatter_plan": (C.c_int, [P, _IP, C.c_int]),
}
_scatter_lib = None

# libmnn_b200_rnn.so (include/mnn_b200_rnn.h): LSTM and RNN, on the runtime and execution handles above
RNN_LIB_PATH = os.path.join(os.path.dirname(LIB_PATH), "libmnn_b200_rnn.so")
RNN_SIGNATURES = {
    "mnnb200_rnn_create": (C.c_int, [P, C.c_int, C.POINTER(P)]),
    "mnnb200_rnn_resize": (C.c_int, [P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "mnnb200_rnn_execute": (C.c_int, [P, P, P, P, P, P, P, P, P, P]),
    "mnnb200_rnn_plan": (C.c_int, [P, _IP, C.c_int]),
}
_rnn_lib = None

# libmnn_b200_grid_sample.so (include/mnn_b200_grid_sample.h): the float GridSample execution, on the runtime and execution handles above
GRID_SAMPLE_LIB_PATH = os.path.join(os.path.dirname(LIB_PATH), "libmnn_b200_grid_sample.so")
GRID_SAMPLE_SIGNATURES = {
    "mnnb200_grid_sample_f32_create": (C.c_int, [P, C.c_int, C.c_int, C.c_int, C.POINTER(P)]),
    "mnnb200_grid_sample_f32_resize": (C.c_int, [P, C.c_int, C.c_int, C.c_int, _IP, _IP]),
    "mnnb200_grid_sample_f32_execute": (C.c_int, [P, P, P, P]),
    "mnnb200_grid_sample_f32_plan": (C.c_int, [P, _IP, C.c_int]),
}
_grid_sample_lib = None

# libmnn_b200_gru.so (include/mnn_b200_gru.h): the GRU execution, on the runtime and execution handles above.  execute's
# params is a host array of 5 * D device pointers
GRU_LIB_PATH = os.path.join(os.path.dirname(LIB_PATH), "libmnn_b200_gru.so")
GRU_SIGNATURES = {
    "mnnb200_gru_create": (C.c_int, [P, C.c_int, C.POINTER(P)]),
    "mnnb200_gru_resize": (C.c_int, [P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "mnnb200_gru_execute": (C.c_int, [P, P, C.POINTER(P), P, P, P]),
    "mnnb200_gru_plan": (C.c_int, [P, _IP, C.c_int]),
}
_gru_lib = None

# libmnn_b200_llm.so (include/mnn_b200_llm.h): MNN-LLM's LayerNorm / RoPE executions, on the runtime and execution handles above
LLM_LIB_PATH = os.path.join(os.path.dirname(LIB_PATH), "libmnn_b200_llm.so")
LLM_SIGNATURES = {
    "mnnb200_layernorm_f32_create": (C.c_int, [P, C.c_int, C.c_float, C.c_int, P, P, C.c_int, C.POINTER(P)]),
    "mnnb200_layernorm_f32_resize": (C.c_int, [P, C.c_int]),
    "mnnb200_layernorm_f32_execute": (C.c_int, [P, P, P, P, P]),
    "mnnb200_rope_f32_create": (C.c_int, [P, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(RopeNorm), C.POINTER(RopeNorm),
                                          C.POINTER(P)]),
    "mnnb200_rope_f32_resize": (C.c_int, [P, C.c_int, C.c_int, C.c_int]),
    "mnnb200_rope_f32_execute": (C.c_int, [P, P, P, P, P, P, P]),
}
_llm_lib = None


def llm_lib():
    """libmnn_b200_llm.so with every LLM_SIGNATURES symbol resolved (after libmnn_b200.so, whose handles it shares)"""
    global _llm_lib
    if _llm_lib is None:
        lib()
        if not os.path.exists(LLM_LIB_PATH):
            raise MnnB200Error(f"{LLM_LIB_PATH} is missing: run `python -m mnn_b200.build` (there is no CPU fallback)")
        L = C.CDLL(LLM_LIB_PATH)
        for name, (res, args) in LLM_SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _llm_lib = L
    return _llm_lib


def deconv_lib():
    """libmnn_b200_deconv.so with every DECONV_SIGNATURES symbol resolved (after libmnn_b200.so, whose handles it shares)"""
    global _deconv_lib
    if _deconv_lib is None:
        lib()
        if not os.path.exists(DECONV_LIB_PATH):
            raise MnnB200Error(f"{DECONV_LIB_PATH} is missing: run `python -m mnn_b200.build` (there is no CPU fallback)")
        L = C.CDLL(DECONV_LIB_PATH)
        for name, (res, args) in DECONV_SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _deconv_lib = L
    return _deconv_lib


def interp_lib():
    """libmnn_b200_interp.so with every INTERP_SIGNATURES symbol resolved (after libmnn_b200.so, whose handles it shares)"""
    global _interp_lib
    if _interp_lib is None:
        lib()
        if not os.path.exists(INTERP_LIB_PATH):
            raise MnnB200Error(f"{INTERP_LIB_PATH} is missing: run `python -m mnn_b200.build` (there is no CPU fallback)")
        L = C.CDLL(INTERP_LIB_PATH)
        for name, (res, args) in INTERP_SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _interp_lib = L
    return _interp_lib


def gather_lib():
    """libmnn_b200_gather.so with every GATHER_SIGNATURES symbol resolved (after libmnn_b200.so, whose handles it shares)"""
    global _gather_lib
    if _gather_lib is None:
        lib()
        if not os.path.exists(GATHER_LIB_PATH):
            raise MnnB200Error(f"{GATHER_LIB_PATH} is missing: run `python -m mnn_b200.build` (there is no CPU fallback)")
        L = C.CDLL(GATHER_LIB_PATH)
        for name, (res, args) in GATHER_SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _gather_lib = L
    return _gather_lib


def scatter_lib():
    """libmnn_b200_scatter.so with every SCATTER_SIGNATURES symbol resolved (after libmnn_b200.so, whose handles it shares)"""
    global _scatter_lib
    if _scatter_lib is None:
        lib()
        if not os.path.exists(SCATTER_LIB_PATH):
            raise MnnB200Error(f"{SCATTER_LIB_PATH} is missing: run `python -m mnn_b200.build` (there is no CPU fallback)")
        L = C.CDLL(SCATTER_LIB_PATH)
        for name, (res, args) in SCATTER_SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _scatter_lib = L
    return _scatter_lib


def rnn_lib():
    """libmnn_b200_rnn.so with every RNN_SIGNATURES symbol resolved (after libmnn_b200.so, whose handles it shares)"""
    global _rnn_lib
    if _rnn_lib is None:
        lib()
        if not os.path.exists(RNN_LIB_PATH):
            raise MnnB200Error(f"{RNN_LIB_PATH} is missing: run `python -m mnn_b200.build` (there is no CPU fallback)")
        L = C.CDLL(RNN_LIB_PATH)
        for name, (res, args) in RNN_SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _rnn_lib = L
    return _rnn_lib


def grid_sample_lib():
    """libmnn_b200_grid_sample.so with every GRID_SAMPLE_SIGNATURES symbol resolved (after libmnn_b200.so, whose handles it shares)"""
    global _grid_sample_lib
    if _grid_sample_lib is None:
        lib()
        if not os.path.exists(GRID_SAMPLE_LIB_PATH):
            raise MnnB200Error(f"{GRID_SAMPLE_LIB_PATH} is missing: run `python -m mnn_b200.build` (there is no CPU fallback)")
        L = C.CDLL(GRID_SAMPLE_LIB_PATH)
        for name, (res, args) in GRID_SAMPLE_SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _grid_sample_lib = L
    return _grid_sample_lib


def gru_lib():
    """libmnn_b200_gru.so with every GRU_SIGNATURES symbol resolved (after libmnn_b200.so, whose handles it shares)"""
    global _gru_lib
    if _gru_lib is None:
        lib()
        if not os.path.exists(GRU_LIB_PATH):
            raise MnnB200Error(f"{GRU_LIB_PATH} is missing: run `python -m mnn_b200.build` (there is no CPU fallback)")
        L = C.CDLL(GRU_LIB_PATH)
        for name, (res, args) in GRU_SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _gru_lib = L
    return _gru_lib


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
