"""Host mirror of the reference's backend plugin surface for the int8 hot path.

Names, argument meaning and error behaviour follow source/core/Backend.hpp / Execution.hpp:
  Runtime.onCreate() -> Backend                         (Backend.hpp:286-409, CUDARuntimeWrapper)
  Backend.onCreate(inputs, outputs, op) -> Execution    (Backend.hpp:89-283; returns None when unsupported, which
                                                         in MNN makes the pipeline fall back -- callers here must
                                                         treat None as an error: there is no CPU fallback)
  Backend.onAcquire / onCopyBuffer / onSync
  Execution.onResize(inputs, outputs) / onExecute(inputs, outputs)   (Execution.hpp:24-135; ErrorCode ints)
Everything below the method signatures goes through the C ABI in include/mnn_b200.h (libmnn_b200.so).
PyTorch is used ONLY as the device-memory / stream plumbing (torch tensors own the HBM buffers).
"""
import ctypes as C
from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np
import torch

from . import _capi
from ._capi import ConvDesc, MnnB200Error, check

NO_ERROR, OUT_OF_MEMORY, NOT_SUPPORT, COMPUTE_SIZE_ERROR, NO_EXECUTION, INVALID_VALUE = 0, 1, 2, 3, 4, 5


def up16(c):
    return (c + 15) // 16 * 16


@dataclass
class QuantAttr:
    """TensorUtils::getQuantInfo order: scale, zero, min, max (source/core/TensorUtils.cpp:940-946)."""
    scale: float = 0.0
    zero: float = 0.0
    min: float = -128.0
    max: float = 127.0


@dataclass
class Tensor:
    """Logical NCHW tensor + device storage.  int8 tensors live as NHWC16, fp32 as NCHW."""
    shape: tuple                       # (n, c, h, w)
    dtype: str = "int8"                # "int8" | "float"
    quant: Optional[QuantAttr] = None
    data: Optional[torch.Tensor] = None

    def ptr(self):
        return C.c_void_p(self.data.data_ptr())


@dataclass
class Op:
    """The slice of MNN::Op the executions need (schema/default/MNN.fbs Convolution2D, QuantizedFloatParam)."""
    type: str                          # ConvInt8 | DepthwiseConvInt8 | FloatToInt8 | Int8ToFloat | LinearW8
    name: str = ""
    conv: Optional[dict] = None        # ic, oc, kernel, stride, pad, dilate, group, relu
    weight: Optional[np.ndarray] = None   # int8 [oc][ic/group][kh][kw]
    wscale: Optional[np.ndarray] = None   # quanParameter.alpha (modern) or symmetricQuan.scale (legacy)
    bias: Optional[np.ndarray] = None     # float (modern) or int32 (legacy)
    wzero: Optional[np.ndarray] = None    # asymmetric weight offsets (LinearW8)
    bits: int = 8                         # LinearW8 weight bits: 4 = weight holds oc * ic / 2 packed nibbles as load() returns them
    legacy: bool = False
    relu6: bool = False
    extra: dict = field(default_factory=dict)


class Runtime:
    """CUDARuntimeWrapper + CUDARuntime: one per GPU, owns/adopts the stream."""

    def __init__(self, device_id: int = 0, adopt_torch_stream: bool = True):
        if not torch.cuda.is_available():
            raise MnnB200Error("mnn_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        torch.cuda.set_device(device_id)
        self.device = torch.device("cuda", device_id)
        self._h = C.c_void_p()
        # torch's DEFAULT stream has handle 0, which the C ABI reads as "create your own (non-blocking) stream" -- torch work on the
        # default stream (fills, copies) would then be UNORDERED with the backend's kernels.  Adopt it as cudaStreamLegacy (0x1)
        # instead: same ordering domain as torch's default stream (graph capture needs a real stream: make one current first).
        stream = None
        if adopt_torch_stream:
            h = torch.cuda.current_stream(self.device).cuda_stream
            stream = C.c_void_p(h if h else 1)
        check(_capi.lib().mnnb200_runtime_create(device_id, stream, C.byref(self._h)), "runtime_create")
        sm = C.c_int()
        major = C.c_int()
        minor = C.c_int()
        mem = C.c_size_t()
        check(_capi.lib().mnnb200_runtime_info(self._h, C.byref(sm), C.byref(major), C.byref(minor), C.byref(mem)))
        self.sm_count, self.cc, self.total_mem = sm.value, (major.value, minor.value), mem.value

    def onCreate(self) -> "Backend":
        return Backend(self)

    def onGabageCollect(self, level=0):
        torch.cuda.empty_cache()

    def __del__(self):
        try:
            if self._h:
                _capi.lib().mnnb200_runtime_destroy(self._h)
                self._h = None
        except Exception:
            pass


class Execution:
    def __init__(self, backend: "Backend"):
        self.backend = backend
        self._h = C.c_void_p()

    def onResize(self, inputs: List[Tensor], outputs: List[Tensor]) -> int:
        return NO_ERROR

    def onExecute(self, inputs: List[Tensor], outputs: List[Tensor]) -> int:
        raise NotImplementedError

    def cost(self):
        b, m = C.c_double(), C.c_double()
        check(_capi.lib().mnnb200_exec_cost(self._h, C.byref(b), C.byref(m)))
        return b.value, m.value

    def __del__(self):
        try:
            if self._h:
                _capi.lib().mnnb200_exec_destroy(self._h)
                self._h = None
        except Exception:
            pass


def _desc(conv):
    kh, kw = conv["kernel"]
    sh, sw = conv.get("stride", (1, 1))
    ph, pw = conv.get("pad", (0, 0))
    dh, dw = conv.get("dilate", (1, 1))
    return ConvDesc(conv["ic"], conv["oc"], kh, kw, sh, sw, ph, pw, dh, dw, conv.get("group", 1),
                    int(bool(conv.get("relu", False))))


def _np_ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class ConvInt8Execution(Execution):
    """ConvInt8CutlassExecution's role with the CPU backend's arithmetic."""

    def __init__(self, backend, op: Op, depthwise=False):
        super().__init__(backend)
        self.op, self.depthwise = op, depthwise
        L = _capi.lib()
        d = _desc(op.conv)
        w = np.ascontiguousarray(op.weight, np.int8)
        ws = np.ascontiguousarray(op.wscale, np.float32)
        rt = backend.runtime._h
        if depthwise:
            b = None if op.bias is None else np.ascontiguousarray(op.bias, np.float32)
            check(L.mnnb200_dwconv_int8_create(rt, C.byref(d), _np_ptr(w), _np_ptr(ws), _np_ptr(b), C.byref(self._h)),
                  "dwconv_int8_create")
        elif op.legacy:
            b = None if op.bias is None else np.ascontiguousarray(op.bias, np.int32)
            check(L.mnnb200_conv_int8_create_legacy(rt, C.byref(d), _np_ptr(w), _np_ptr(ws), _np_ptr(b),
                                                    C.byref(self._h)), "conv_int8_create_legacy")
        else:
            b = None if op.bias is None else np.ascontiguousarray(op.bias, np.float32)
            check(L.mnnb200_conv_int8_create(rt, C.byref(d), _np_ptr(w), _np_ptr(ws), _np_ptr(b), C.byref(self._h)),
                  "conv_int8_create")

    def set_variant(self, v):
        check(_capi.lib().mnnb200_conv_int8_set_variant(self._h, v))

    def onResize(self, inputs, outputs):
        x, y = inputs[0], outputs[0]
        n, _, ih, iw = x.shape
        qi, qo = x.quant or QuantAttr(), y.quant or QuantAttr()
        known = len(y.shape) == 4 and y.shape[2] > 0 and y.shape[3] > 0 and self.op.extra.get("shape_known")
        oh, ow = C.c_int(y.shape[2] if known else 0), C.c_int(y.shape[3] if known else 0)
        f = _capi.lib().mnnb200_dwconv_int8_resize if self.depthwise else _capi.lib().mnnb200_conv_int8_resize
        st = f(self._h, n, ih, iw, qi.scale, int(qi.zero), qo.scale, int(qo.zero), int(qo.min), int(qo.max),
               C.byref(oh), C.byref(ow))
        if st == 0:
            y.shape = (n, self.op.conv["oc"], oh.value, ow.value)
        return st

    def onExecute(self, inputs, outputs):
        f = _capi.lib().mnnb200_dwconv_int8_execute if self.depthwise else _capi.lib().mnnb200_conv_int8_execute
        return f(self._h, inputs[0].ptr(), outputs[0].ptr())


class ConvGroupExecution(Execution):
    """One persistent launch for a list of GEMM-shaped ConvInt8Executions whose inputs are all ready when the group is
    enqueued (mnnb200_conv_group_*): the role of Pipeline::execute's per-command walk for that run of commands."""

    def __init__(self, backend, members: List[ConvInt8Execution]):
        super().__init__(backend)
        self.members = list(members)          # keeps the member executions alive
        arr = (C.c_void_p * len(members))(*[m._h for m in members])
        check(_capi.lib().mnnb200_conv_group_create(backend.runtime._h, arr, len(members), C.byref(self._h)),
              "conv_group_create")

    @staticmethod
    def groupable(ex) -> bool:
        return isinstance(ex, ConvInt8Execution) and not ex.depthwise and bool(_capi.lib().mnnb200_conv_int8_groupable(ex._h))

    def bind(self, xs: List[Tensor], ys: List[Tensor]) -> int:
        n = len(self.members)
        ax = (C.c_void_p * n)(*[x.data.data_ptr() for x in xs])
        ay = (C.c_void_p * n)(*[y.data.data_ptr() for y in ys])
        return _capi.lib().mnnb200_conv_group_bind(self._h, ax, ay)

    def onExecute(self, inputs=None, outputs=None):
        return _capi.lib().mnnb200_conv_group_execute(self._h)

    def launches(self) -> int:
        """kernel launches per execute: one per kernel that runs a member (the last field of mnnb200_conv_int8_group_plan)"""
        kernels = set()
        for m in self.members:
            f = (C.c_int * 11)()
            check(_capi.lib().mnnb200_conv_int8_group_plan(m._h, f, 11), "conv_int8_group_plan")
            kernels.add(f[10])
        return len(kernels)


def encode_winograd_attr(units):
    """WinogradInt8Attr::encode (source/core/WinogradInt8Attr.hpp:45-63): units = [(kyStart, kxStart, kernelY, kernelX,
    unitY, unitX, inputScales[a2], inputZeroPoints[a2], weightScales[a2*oc])] -> the int32 blob stored in
    Convolution2D.symmetricQuan.winogradAttr."""
    out = [0, len(units)]
    for (ky0, kx0, ky, kx, uy, ux, ins, inz, ws) in units:
        body = np.concatenate([np.asarray([ky0, kx0, ky, kx, uy, ux], np.int32),
                               np.ascontiguousarray(ins, np.float32).ravel().view(np.int32),
                               np.ascontiguousarray(inz, np.int32).ravel(),
                               np.ascontiguousarray(ws, np.float32).ravel().view(np.int32)])
        out += [body.size] + body.tolist()
    return np.asarray(out, np.int32)


class ConvInt8WinogradExecution(Execution):
    """ConvInt8Winograd (source/backend/cpu/compute/ConvInt8Winograd.cpp): op.extra['winograd_attr'] is the op's
    symmetricQuan.winogradAttr blob, passed to the library verbatim."""

    def __init__(self, backend, op: Op):
        super().__init__(backend)
        self.op = op
        d = _desc(op.conv)
        w = np.ascontiguousarray(op.weight, np.int8)
        ws = np.ascontiguousarray(op.wscale, np.float32)
        b = None if op.bias is None else np.ascontiguousarray(op.bias, np.float32)
        attr = np.ascontiguousarray(op.extra["winograd_attr"], np.int32)
        check(_capi.lib().mnnb200_conv_int8_wino_create(backend.runtime._h, C.byref(d), _np_ptr(w), _np_ptr(ws), _np_ptr(b),
                                                        _np_ptr(attr), int(attr.size), C.byref(self._h)),
              "conv_int8_wino_create")

    def onResize(self, inputs, outputs):
        x, y = inputs[0], outputs[0]
        n, _, ih, iw = x.shape
        qi, qo = x.quant or QuantAttr(), y.quant or QuantAttr()
        oh, ow = C.c_int(0), C.c_int(0)
        st = _capi.lib().mnnb200_conv_int8_wino_resize(self._h, n, ih, iw, qi.scale, int(qi.zero), qo.scale, int(qo.zero),
                                                       int(qo.min), int(qo.max), C.byref(oh), C.byref(ow))
        if st == 0:
            y.shape = (n, self.op.conv["oc"], oh.value, ow.value)
        return st

    def onExecute(self, inputs, outputs):
        return _capi.lib().mnnb200_conv_int8_wino_execute(self._h, inputs[0].ptr(), outputs[0].ptr())


class FloatToInt8Execution(Execution):
    def onExecute(self, inputs, outputs):
        x, y = inputs[0], outputs[0]
        n, c, h, w = x.shape
        q = y.quant
        return _capi.lib().mnnb200_float_to_int8(self.backend.runtime._h, x.ptr(), n, c, h, w, q.scale, q.zero,
                                                 int(q.min), int(q.max), y.ptr())


class Int8ToFloatExecution(Execution):
    def onExecute(self, inputs, outputs):
        x, y = inputs[0], outputs[0]
        n, c, h, w = x.shape
        q = x.quant
        return _capi.lib().mnnb200_int8_to_float(self.backend.runtime._h, x.ptr(), n, c, h, w, q.scale, q.zero, y.ptr())


class BinaryAddInt8Execution(Execution):
    """BinaryOp ADD on int8 tensors (CPUBinaryInt8 / execution/int8/BinaryInt8Execution.cu)."""

    def onExecute(self, inputs, outputs):
        a, b, y = inputs[0], inputs[1], outputs[0]
        n, c, h, w = y.shape
        qa, qb, qy = a.quant, b.quant, y.quant
        return _capi.lib().mnnb200_binary_add_int8(self.backend.runtime._h, a.ptr(), qa.scale, int(qa.zero), b.ptr(), qb.scale,
                                                   int(qb.zero), y.ptr(), qy.scale, int(qy.zero), int(qy.min), int(qy.max),
                                                   n, c, h, w)


class AvgPoolInt8Execution(Execution):
    """Pooling AVE between int8 tensors (quant attrs may differ: float pooling bracketed by casts, fused)."""

    def __init__(self, backend, op):
        super().__init__(backend)
        self.a = op.extra

    def onResize(self, inputs, outputs):
        from .graph import float_pool_params      # ShapePool + CPUPool resolution (ceilModel, pads, SAME/VALID, global)
        n, c, h, w = inputs[0].shape
        oh, ow, self.k, self.s, self.p, self.pt = float_pool_params(h, w, self.a)
        outputs[0].shape = (n, c, oh, ow)
        return NO_ERROR

    def onExecute(self, inputs, outputs):
        x, y = inputs[0], outputs[0]
        n, c, h, w = x.shape
        qi, qo = x.quant, y.quant
        return _capi.lib().mnnb200_avgpool_int8(self.backend.runtime._h, x.ptr(), n, c, h, w, self.k[0], self.k[1], self.s[0],
                                                self.s[1], self.p[0], self.p[1], self.pt, self.a.get("count_type", 0),
                                                qi.scale, qi.zero, qo.scale, qo.zero, int(qo.min), int(qo.max), y.ptr(),
                                                y.shape[2], y.shape[3])


class ScaleInt8Execution(Execution):
    """Scale between int8 tensors (CPUScaleInt8): op.extra = {scale: [c], bias: [c] or None}."""

    def __init__(self, backend, op):
        super().__init__(backend)
        sc = np.ascontiguousarray(op.extra["scale"], np.float32)
        bi = None if op.extra.get("bias") is None else np.ascontiguousarray(op.extra["bias"], np.float32)
        check(_capi.lib().mnnb200_scale_int8_create(backend.runtime._h, int(sc.size), _np_ptr(sc), _np_ptr(bi), C.byref(self._h)),
              "scale_int8_create")

    def onResize(self, inputs, outputs):
        qi, qo = inputs[0].quant, outputs[0].quant
        outputs[0].shape = inputs[0].shape
        return _capi.lib().mnnb200_scale_int8_resize(self._h, qi.scale, int(qi.zero), qo.scale, int(qo.zero), int(qo.min), int(qo.max))

    def onExecute(self, inputs, outputs):
        n, c, h, w = inputs[0].shape
        return _capi.lib().mnnb200_scale_int8_execute(self._h, inputs[0].ptr(), n, h, w, outputs[0].ptr())


class PoolInt8Execution(Execution):
    """Pooling between int8 tensors with EQUAL quant attrs (CPUPoolInt8, x86 semantics): op.extra = pool attrs + is_avg."""

    def __init__(self, backend, op):
        super().__init__(backend)
        self.a = op.extra

    def onResize(self, inputs, outputs):
        from .graph import pool_out_and_pad
        n, c, h, w = inputs[0].shape
        a = self.a
        if a.get("is_global"):
            self.k, self.s, self.p, oh, ow = (h, w), (h, w), (0, 0), 1, 1
        else:
            oh, ow, ph, pw = pool_out_and_pad(h, w, a)
            self.k, self.s, self.p = a["kernel"], a["stride"], (ph, pw)
        outputs[0].shape = (n, c, oh, ow)
        return NO_ERROR

    def onExecute(self, inputs, outputs):
        n, c, h, w = inputs[0].shape
        y = outputs[0]
        return _capi.lib().mnnb200_pool_int8(self.backend.runtime._h, inputs[0].ptr(), n, c, h, w, self.k[0], self.k[1], self.s[0],
                                             self.s[1], self.p[0], self.p[1], int(bool(self.a.get("is_avg", True))), y.ptr(),
                                             y.shape[2], y.shape[3])


class SoftmaxInt8Execution(Execution):
    def onExecute(self, inputs, outputs):
        x, y = inputs[0], outputs[0]
        rows, c = x.shape[0], x.shape[1]
        qi, qo = x.quant, y.quant
        return _capi.lib().mnnb200_softmax_int8(self.backend.runtime._h, x.ptr(), rows, c, qi.scale, qi.zero, qo.scale, qo.zero,
                                                int(qo.min), int(qo.max), y.ptr())


class LinearW8Execution(Execution):
    """Conv1x1 with int8 weights + dynamic activation quantisation (the MNN-LLM linear layer)."""

    def __init__(self, backend, op: Op):
        super().__init__(backend)
        al = np.ascontiguousarray(op.wscale, np.float32)
        wz = None if op.wzero is None else np.ascontiguousarray(op.wzero, np.float32)
        b = None if op.bias is None else np.ascontiguousarray(op.bias, np.float32)
        relu = int(bool(op.conv.get("relu", False)))
        ic, self.oc = op.conv["ic"], op.conv["oc"]
        # alpha [oc] (per channel) or [oc, blocks] (K-blocked weight scales, quant_block), wzero of the same shape or None
        blocks = al.shape[1] if al.ndim == 2 else 1
        if op.bits == 4:
            w = np.ascontiguousarray(op.weight, np.uint8).reshape(-1)
            if w.size * 2 != self.oc * ic:
                raise MnnB200Error(f"LinearW8 bits=4: {w.size} packed bytes for oc {self.oc} x ic {ic}")
            create = _capi.lib().mnnb200_linear_w4_create_blocked
        elif op.bits == 8:
            w = np.ascontiguousarray(op.weight, np.int8).reshape(self.oc, ic)
            create = _capi.lib().mnnb200_linear_w8_create_blocked
        else:
            raise MnnB200Error(f"LinearW8: {op.bits}-bit weights are not supported")
        check(create(backend.runtime._h, ic, self.oc, blocks, _np_ptr(w), _np_ptr(al), _np_ptr(wz), _np_ptr(b), relu,
                     int(op.relu6), C.byref(self._h)), f"LinearW8 bits={op.bits}")

    def onResize(self, inputs, outputs):
        tokens = inputs[0].shape[0]
        st = _capi.lib().mnnb200_linear_w8_resize(self._h, tokens)
        if st == 0:
            outputs[0].shape = (tokens, self.oc)
        return st

    def onExecute(self, inputs, outputs):
        return _capi.lib().mnnb200_linear_w8_execute(self._h, inputs[0].ptr(), outputs[0].ptr())


class MatMulExecution(Execution):
    """MatMul / BatchMatMul on float tensors (MatMulExecution.cu's role): C = op(A) op(B) (+ bias) over the batch dims
    ShapeMatMul broadcasts (right-aligned, a dim of 1 against any size), with its squeeze of a 1-D operand: A of [l] is one
    row, B of [l] one column (their transpose flags ignored), and the output drops that dim.  fp32 operands run through
    mnnb200_matmul_create_broadcast; fp16 operands (the f16 kernel) through mnnb200_matmul_create, without broadcast.
    op.extra: transpose_a, transpose_b."""

    def __init__(self, backend, op: Op):
        super().__init__(backend)
        self.ta, self.tb = int(bool(op.extra.get("transpose_a", False))), int(bool(op.extra.get("transpose_b", False)))
        self.bias = None if op.bias is None else torch.from_numpy(np.ascontiguousarray(op.bias, np.float32)).to(backend.runtime.device)

    def onResize(self, inputs, outputs):
        a, b = inputs[0], inputs[1]
        sa, sb = tuple(int(v) for v in a.shape), tuple(int(v) for v in b.shape)
        if len(sa) < 1 or len(sb) < 1:
            return NOT_SUPPORT
        ta, tb = int(len(sa) > 1 and self.ta), int(len(sb) == 1 or self.tb)   # B of [l] is K-major [h = 1][l]
        e, l = (1, sa[0]) if len(sa) == 1 else (sa[-1], sa[-2]) if ta else (sa[-2], sa[-1])
        h, l2 = (1, sb[0]) if len(sb) == 1 else (sb[-2], sb[-1]) if tb else (sb[-1], sb[-2])
        if l != l2:
            return COMPUTE_SIZE_ERROR
        nd = max(len(sa), len(sb), 2) - 2
        if nd > 8:
            return NOT_SUPPORT
        ad = (1,) * (nd - max(len(sa) - 2, 0)) + sa[:-2]
        bd = (1,) * (nd - max(len(sb) - 2, 0)) + sb[:-2]
        if any(x != y and x != 1 and y != 1 for x, y in zip(ad, bd)):
            return NOT_SUPPORT
        cd = tuple(y if x == 1 else x for x, y in zip(ad, bd))
        f16 = a.data is not None and a.data.dtype == torch.float16
        if f16 and ad != bd:
            return NOT_SUPPORT
        if self._h:
            _capi.lib().mnnb200_exec_destroy(self._h)
            self._h = C.c_void_p()
        L = _capi.lib()
        if f16:
            st = L.mnnb200_matmul_create(self.backend.runtime._h, int(np.prod(cd, dtype=np.int64)), e, l, h, ta, tb, 1,
                                         C.byref(self._h))
        else:
            def arr(v):
                return (C.c_int * max(len(v), 1))(*v)
            st = L.mnnb200_matmul_create_broadcast(self.backend.runtime._h, nd, arr(cd), arr(ad), arr(bd), e, l, h, ta, tb,
                                                   C.byref(self._h))
        if st == 0:
            outputs[0].shape = cd + ((e,) if len(sa) > 1 else ()) + ((h,) if len(sb) > 1 else ()) or (1,)
        return st

    def onExecute(self, inputs, outputs):
        return _capi.lib().mnnb200_matmul_execute(self._h, inputs[0].ptr(), inputs[1].ptr(),
                                                  None if self.bias is None else C.c_void_p(self.bias.data_ptr()), outputs[0].ptr())


class ConvF32Execution(Execution):
    """Float Convolution (any group, split-TF32 wgmma) or ConvolutionDepthwise on NCHW fp32 tensors: the CPU backend's float
    convolutions.  op.weight fp32 [oc][ic/group][kh][kw], op.bias fp32 [oc] or None; op.conv['relu'] / op.relu6."""

    def __init__(self, backend, op: Op, depthwise=False):
        super().__init__(backend)
        self.op, self.depthwise = op, depthwise
        d = _desc(op.conv)
        w = np.ascontiguousarray(op.weight, np.float32)
        b = None if op.bias is None else np.ascontiguousarray(op.bias, np.float32)
        L = _capi.lib()
        f, name = ((L.mnnb200_dwconv_f32_create, "dwconv_f32_create") if depthwise else
                   (L.mnnb200_conv_f32_create_grouped, "conv_f32_create_grouped") if d.group > 1 else
                   (L.mnnb200_conv_f32_create, "conv_f32_create"))
        check(f(backend.runtime._h, C.byref(d), _np_ptr(w), _np_ptr(b), int(op.relu6), C.byref(self._h)), name)

    def onResize(self, inputs, outputs):
        n, _, ih, iw = inputs[0].shape
        oh, ow = C.c_int(0), C.c_int(0)
        f = _capi.lib().mnnb200_dwconv_f32_resize if self.depthwise else _capi.lib().mnnb200_conv_f32_resize
        st = f(self._h, n, ih, iw, C.byref(oh), C.byref(ow))
        if st == 0:
            outputs[0].shape = (n, self.op.conv["oc"], oh.value, ow.value)
        return st

    def onExecute(self, inputs, outputs):
        f = _capi.lib().mnnb200_dwconv_f32_execute if self.depthwise else _capi.lib().mnnb200_conv_f32_execute
        return f(self._h, inputs[0].ptr(), outputs[0].ptr())


class DeconvF32Execution(Execution):
    """Float Deconvolution (group 1, split-TF32 wgmma over the stride phases) or DeconvolutionDepthwise on NCHW fp32 tensors: the
    CPU backend's CPUDeconvolution / CPUDeconvolutionDepthwise.  op.weight fp32 [ic][oc][kh][kw] ([c][1][kh][kw] depthwise),
    op.bias fp32 [oc] or None; op.conv['pad'] the begin pads, op.conv['out_hw'] an explicit output size (else the natural one)."""

    def __init__(self, backend, op: Op, depthwise=False):
        super().__init__(backend)
        self.op, self.depthwise = op, depthwise
        d = _desc(op.conv)
        w = np.ascontiguousarray(op.weight, np.float32)
        b = None if op.bias is None else np.ascontiguousarray(op.bias, np.float32)
        f = _capi.deconv_lib().mnnb200_dwdeconv_f32_create if depthwise else _capi.deconv_lib().mnnb200_deconv_f32_create
        check(f(backend.runtime._h, C.byref(d), _np_ptr(w), _np_ptr(b), int(op.relu6), C.byref(self._h)),
              "dwdeconv_f32_create" if depthwise else "deconv_f32_create")

    def onResize(self, inputs, outputs):
        n, _, ih, iw = inputs[0].shape
        oh, ow = (C.c_int(v) for v in self.op.conv.get("out_hw", (0, 0)))
        f = _capi.deconv_lib().mnnb200_dwdeconv_f32_resize if self.depthwise else _capi.deconv_lib().mnnb200_deconv_f32_resize
        st = f(self._h, n, ih, iw, C.byref(oh), C.byref(ow))
        if st == 0:
            outputs[0].shape = (n, self.op.conv["oc"], oh.value, ow.value)
        return st

    def onExecute(self, inputs, outputs):
        f = _capi.deconv_lib().mnnb200_dwdeconv_f32_execute if self.depthwise else _capi.deconv_lib().mnnb200_deconv_f32_execute
        return f(self._h, inputs[0].ptr(), outputs[0].ptr())


class InterpF32Execution(Execution):
    """Float Interp on NCHW fp32 tensors: the CPU backend's CPUInterp as the geometry stage leaves it.  op.extra: resize_type (1
    nearest, 2 bilinear, 3 cubic, 4 nearest-round), scale (h, w), offset (h, w) -- the lowered op's coordinate transform, src =
    dst * scale + offset -- and out_hw, the output size."""

    def __init__(self, backend, op: Op):
        super().__init__(backend)
        self.op = op
        e = op.extra
        (hs, ws), (ho, wo) = e["scale"], e.get("offset", (0.0, 0.0))
        check(_capi.interp_lib().mnnb200_interp_f32_create(backend.runtime._h, int(e["resize_type"]), ws, hs, wo, ho,
                                                           C.byref(self._h)), "interp_f32_create")

    def onResize(self, inputs, outputs):
        n, c, ih, iw = inputs[0].shape
        oh, ow = self.op.extra["out_hw"]
        st = _capi.interp_lib().mnnb200_interp_f32_resize(self._h, n * c, ih, iw, oh, ow)
        if st == 0:
            outputs[0].shape = (n, c, oh, ow)
        return st

    def onExecute(self, inputs, outputs):
        return _capi.interp_lib().mnnb200_interp_f32_execute(self._h, inputs[0].ptr(), outputs[0].ptr())


class GatherExecution(Execution):
    """Gather / GatherV2 / GatherND / GatherElements on 4-byte tensors (fp32 or int32) with int32 indices, shapes as given (any
    rank): the CPU backend's While loops of GeometryGather.cpp.  op.type: "Gather" (GatherV2 alike), "GatherND" or
    "GatherElements"; op.extra["axis"]: the Gather / GatherElements axis or GatherND's batch dims (default 0).  The output's
    shape is set at onResize."""

    MODES = {"Gather": 0, "GatherND": 1, "GatherElements": 2}

    def __init__(self, backend, op: Op):
        super().__init__(backend)
        self.op = op
        self.mode = self.MODES[op.type]
        check(_capi.gather_lib().mnnb200_gather_create(backend.runtime._h, self.mode, C.byref(self._h)), "gather_create")

    def onResize(self, inputs, outputs):
        p, i = tuple(inputs[0].shape), tuple(inputs[1].shape) or (1,)
        axis = int(self.op.extra.get("axis", 0))
        ints = lambda v: (C.c_int * len(v))(*v)   # noqa: E731
        st = _capi.gather_lib().mnnb200_gather_resize(self._h, ints(p), len(p), ints(i), len(i), axis)
        if st == 0:
            if self.mode == 0:
                a = axis % len(p)
                outputs[0].shape = p[:a] + tuple(inputs[1].shape) + p[a + 1:]
            elif self.mode == 1:
                outputs[0].shape = i[:-1] + p[axis + i[-1]:]
            else:
                outputs[0].shape = i
        return st

    def onExecute(self, inputs, outputs):
        return _capi.gather_lib().mnnb200_gather_execute(self._h, inputs[0].ptr(), inputs[1].ptr(), outputs[0].ptr())


class Backend:
    """CUDABackend's role: creator map, buffer acquisition, host<->device copies with layout + quant casts."""

    _creators = {}

    def __init__(self, runtime: Runtime):
        self.runtime = runtime

    @classmethod
    def addCreator(cls, op_type, fn):  # CUDABackend::addCreator
        cls._creators[op_type] = fn

    def onCreate(self, inputs, outputs, op: Op) -> Optional[Execution]:
        fn = self._creators.get(op.type)
        return fn(self, inputs, outputs, op) if fn else None

    def onAcquire(self, t: Tensor) -> Tensor:
        dev = self.runtime.device
        if t.dtype == "int8":
            n, c, h, w = t.shape
            t.data = torch.zeros((n, h, w, up16(c)), dtype=torch.int8, device=dev)
        else:
            t.data = torch.zeros(t.shape, dtype=torch.float32, device=dev)
        return t

    def onCopyBuffer(self, src, dst):
        """host numpy (NCHW) <-> device Tensor, with the layout change and, when types differ, the quant cast."""
        L, rt = _capi.lib(), self.runtime._h
        if isinstance(src, np.ndarray):          # host -> device
            n, c, h, w = dst.shape
            if dst.dtype == "float":
                dst.data.copy_(torch.from_numpy(np.ascontiguousarray(src, np.float32)).reshape(dst.shape))
            elif src.dtype == np.int8:
                stage = torch.from_numpy(np.ascontiguousarray(src)).to(self.runtime.device)
                check(L.mnnb200_pack_nchw_int8(rt, C.c_void_p(stage.data_ptr()), n, c, h, w, dst.ptr()), "pack")
            else:                                # float host -> int8 device: FloatToInt8 inside the copy
                stage = torch.from_numpy(np.ascontiguousarray(src, np.float32)).to(self.runtime.device)
                q = dst.quant
                check(L.mnnb200_float_to_int8(rt, C.c_void_p(stage.data_ptr()), n, c, h, w, q.scale, q.zero,
                                              int(q.min), int(q.max), dst.ptr()), "float_to_int8")
            return None
        n, c, h, w = src.shape                   # device -> host
        want = dst if isinstance(dst, str) else "same"
        if src.dtype == "float":
            return src.data.cpu().numpy()
        if want == "float":                      # dequantise inside the copy (CUDABackend.cpp:537-589)
            out = torch.empty((n, c, h, w), dtype=torch.float32, device=self.runtime.device)
            q = src.quant
            check(L.mnnb200_int8_to_float(rt, src.ptr(), n, c, h, w, q.scale, q.zero, C.c_void_p(out.data_ptr())))
            return out.cpu().numpy()
        out = torch.empty((n, c, h, w), dtype=torch.int8, device=self.runtime.device)
        check(L.mnnb200_unpack_nchw_int8(rt, src.ptr(), n, c, h, w, C.c_void_p(out.data_ptr())), "unpack")
        return out.cpu().numpy()

    def onSync(self):
        check(_capi.lib().mnnb200_runtime_sync(self.runtime._h), "sync")


def _create_conv_int8(b, i, o, op):
    if op.conv.get("group", 1) != 1:
        return None
    if op.extra.get("winograd_attr") is not None:     # ConvInt8Winograd::mustUse, CPUConvolution.cpp:336-339
        return ConvInt8WinogradExecution(b, op)
    return ConvInt8Execution(b, op)


Backend.addCreator("ConvInt8", _create_conv_int8)
Backend.addCreator("DepthwiseConvInt8", lambda b, i, o, op: ConvInt8Execution(b, op, depthwise=True))
Backend.addCreator("FloatToInt8", lambda b, i, o, op: FloatToInt8Execution(b))
Backend.addCreator("Int8ToFloat", lambda b, i, o, op: Int8ToFloatExecution(b))
Backend.addCreator("BinaryAddInt8", lambda b, i, o, op: BinaryAddInt8Execution(b))
Backend.addCreator("AvgPoolInt8", lambda b, i, o, op: AvgPoolInt8Execution(b, op))
Backend.addCreator("ScaleInt8", lambda b, i, o, op: ScaleInt8Execution(b, op))
Backend.addCreator("PoolInt8", lambda b, i, o, op: PoolInt8Execution(b, op))
Backend.addCreator("SoftmaxInt8", lambda b, i, o, op: SoftmaxInt8Execution(b))
Backend.addCreator("MatMul", lambda b, i, o, op: MatMulExecution(b, op))
Backend.addCreator("BatchMatMul", lambda b, i, o, op: MatMulExecution(b, op))
Backend.addCreator("LinearW8", lambda b, i, o, op: LinearW8Execution(b, op))


def _create_conv_f32(b, i, o, op):
    c, g = op.conv, op.conv.get("group", 1)
    kh, kw = c.get("kernel", (1, 1))
    if g < 1 or c["ic"] % g or c["oc"] % g or np.size(op.weight) != c["oc"] * (c["ic"] // g) * kh * kw:
        return None                       # weights not shaped [oc][ic/group][kh][kw]
    return ConvF32Execution(b, op)


Backend.addCreator("Convolution", _create_conv_f32)
Backend.addCreator("ConvolutionDepthwise", lambda b, i, o, op: ConvF32Execution(b, op, depthwise=True))


def _create_deconv_f32(b, i, o, op):
    if op.conv.get("group", 1) != 1:      # CPUDeconvolution ignores group; a grouped deconvolution is not taken
        return None
    return DeconvF32Execution(b, op)


Backend.addCreator("DeconvF32", _create_deconv_f32)
Backend.addCreator("DwDeconvF32", lambda b, i, o, op: DeconvF32Execution(b, op, depthwise=True))
Backend.addCreator("InterpF32", lambda b, i, o, op: InterpF32Execution(b, op))
for _t in ("Gather", "GatherND", "GatherElements"):
    Backend.addCreator(_t, lambda b, i, o, op: GatherExecution(b, op))
