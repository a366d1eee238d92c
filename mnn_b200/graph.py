"""Shape propagation over a parsed .mnn graph for the op set of the int8 CNN path
(the slice of source/shape/ShapeConvolution.cpp, ShapePool.cpp, ShapeBinaryOp.cpp ... the path needs)."""
from typing import Dict, List

from .mnn_file import Net, OpNode


def conv_out_and_pad(i, k, s, d, pad, pad_mode):
    """ConvolutionCommon::convolutionPad + ShapeConvolution (source/core/ConvolutionCommon.cpp:944-990,
    source/shape/ShapeConvolution.cpp): SAME => out = ceil(i/s), pad_begin = max(0, (out-1)*s + kd - i) / 2."""
    kd = d * (k - 1) + 1
    if pad_mode == 2:  # SAME
        o = (i + s - 1) // s
        need = max(0, (o - 1) * s + kd - i)
        return o, need // 2
    if pad_mode == 1:  # VALID
        return (i - kd) // s + 1, 0
    return (i + 2 * pad - kd) // s + 1, pad


def pool_out_and_pad(h, w, a):
    """ShapePool (source/shape/ShapePool.cpp:38-77) + the begin pads CPUPool resolves (CPUPool.cpp:45-75).
    Returns (oh, ow, pad_h_begin, pad_w_begin)."""
    kh, kw = a["kernel"]
    sh, sw = a["stride"]
    ph, pw = a.get("pad", (0, 0))
    pads = a.get("pads")
    hh, ww = h, w
    if pads is not None and len(pads) == 2:
        hh += pads[0] + pads[1]
    elif pads is not None and len(pads) == 4:
        ww += pads[1] + pads[3]
        hh += pads[0] + pads[2]
    else:
        hh += 2 * ph
        ww += 2 * pw
    kh, kw = min(kh, hh), min(kw, ww)
    pt = a.get("pad_type", 0)
    if pt == 2:      # SAME
        oh, ow = -(-hh // sh), -(-ww // sw)
        return oh, ow, max(0, (oh - 1) * sh + kh - h) // 2, max(0, (ow - 1) * sw + kw - w) // 2
    if pt == 1:      # VALID
        return -(-(hh - kh + 1) // sh), -(-(ww - kw + 1) // sw), 0, 0
    if a.get("ceil_model", True):
        oh, ow = -(-(hh - kh) // sh) + 1, -(-(ww - kw) // sw) + 1
    else:
        oh, ow = (hh - kh) // sh + 1, (ww - kw) // sw + 1
    if pads is not None and len(pads) == 4:
        ph, pw = pads[0], pads[1]
    return oh, ow, ph, pw


def float_pool_params(h, w, a):
    """What CPUPool::onResize (CPUPool.cpp:25-75) hands to the float pooling functions:
    -> (oh, ow, kernel, stride, begin pads, pad type).  Unlike CPUPoolInt8 it keeps the op's kernel unclamped, also in the
    SAME pad; and a CAFFE pool that carries a `pads` vector, of any length, runs as VALID, so that DEFAULT counting
    excludes the padding."""
    pt = a.get("pad_type", 0)
    if a.get("is_global"):
        return 1, 1, (h, w), (h, w), (0, 0), pt
    oh, ow, ph, pw = pool_out_and_pad(h, w, a)
    (kh, kw), (sh, sw) = a["kernel"], a["stride"]
    if pt == 2:
        ph, pw = max(0, (oh - 1) * sh + kh - h) // 2, max(0, (ow - 1) * sw + kw - w) // 2
    if pt == 0 and a.get("pads") is not None:
        pt = 1
    return oh, ow, (kh, kw), (sh, sw), (ph, pw), pt


def infer_shapes(net: Net, input_shape) -> Dict[int, tuple]:
    shapes: Dict[int, tuple] = {}
    for op in net.ops:
        ins = [shapes.get(i) for i in op.inputs]
        if op.type == "Input":
            shapes[op.outputs[0]] = tuple(input_shape)
        elif op.type in ("Convolution", "ConvolutionDepthwise", "ConvInt8", "DepthwiseConvInt8"):
            n, _, h, w = ins[0]
            c = op.conv
            oh, ph = conv_out_and_pad(h, c.kernel[0], c.stride[0], c.dilate[0], c.pad[0], c.pad_mode)
            ow, pw = conv_out_and_pad(w, c.kernel[1], c.stride[1], c.dilate[1], c.pad[1], c.pad_mode)
            op.attrs["resolved_pad"] = (ph, pw)
            op.attrs["in_shape"] = ins[0]
            shapes[op.outputs[0]] = (n, c.oc, oh, ow)
        elif op.type == "Pooling":
            n, c, h, w = ins[0]
            a = op.attrs
            if a.get("is_global"):
                shapes[op.outputs[0]] = (n, c, 1, 1)
            else:
                oh, ow, ph, pw = pool_out_and_pad(h, w, a)
                a["resolved_pad"] = (ph, pw)
                shapes[op.outputs[0]] = (n, c, oh, ow)
        elif op.type in ("BinaryOp", "Eltwise", "ReLU", "ReLU6", "Softmax", "FloatToInt8", "Int8ToFloat", "Scale"):
            shapes[op.outputs[0]] = ins[0]
        elif op.type == "ConvertTensor":
            shapes[op.outputs[0]] = ins[0]      # logical NCHW bookkeeping only; layout is the backend's business
        elif op.type == "Squeeze":
            s = ins[0]
            shapes[op.outputs[0]] = (s[0], s[1]) if len(s) == 4 and s[2] == 1 and s[3] == 1 else s
        elif op.type == "Shape":
            shapes[op.outputs[0]] = (len(ins[0]),)
        elif op.type == "Reshape":
            s = ins[0]
            tot = 1
            for v in s:
                tot *= v
            shapes[op.outputs[0]] = (s[0], tot // s[0])
        else:
            raise NotImplementedError(f"shape inference: {op.type}")
    return shapes


def dense_convs(net: Net) -> List[OpNode]:
    return [op for op in net.ops if op.type in ("Convolution", "ConvInt8") and op.conv.group == 1]
