"""Restatement of the reference CPU's fp32 Interp (and of Resize, which the geometry stage lowers to a bilinear Interp).

Finding (the live reference, x86 with AVX2 / AVX512): the CPU runtime's main backend there is AVX2Backend, which packs float
NC4HW4 by 8 or 16 and creates only the ops OpCommonUtils::opCompabilityForLowp lists (AVX2Backend.cpp:317-334).  Interp is not
among them, so every Interp of an MNN_FORWARD_CPU session runs on the pack-4 backup CPUBackend: CPUInterp over
CPUResize.hpp's C4 loops and compute/ResizeFunction.cpp's SSE Vec4 sample / line functions (compute/ is built without -mfma:
every product and sum is rounded on its own).  The layout conversions between the two packs move values without changing
them, so the recorded outputs are exactly what that code computes; tests/golden/interp_f32_golden.npz, recorded through
oracle/refdump_interp.cpp, equals this restatement bit for bit.

transform() restates _ConverterInterp (source/geometry/ConvertUtils.hpp) as GeometryImageOp calls it: the op's ctm,
alignCorners and halfPixelCenters, the input / output sizes, or a float scales input (then scale = 1 / the factor and only the
offsets are derived).  interp() restates CPUInterp per resize type in numpy float32, one rounded operation at a time, the cubic
weights in float64 where the CPU computes them in double; interp64() is the same resampling in float64 throughout, for a sanity
bound."""
import json
import os
import struct
import subprocess
import tempfile

import numpy as np

F = np.float32
CTM = {"NotSet": 0, "AlignCorners": 1, "HalfPixels": 2, "PytorchHalfPixels": 3, "Asymmetric": 4, "TensorflowHalfPixels": 5,
       "TensorflowCropAndResize": 6}


def transform(resize_type, ctm, align_corners, half_pixel, in_hw, out_hw, scales=None):
    """(width_scale, height_scale, width_offset, height_offset) as float32, as the geometry writes them into the lowered Interp.
    ctm: a CTM name or value; scales: (height factor, width factor) of a float scales input, or None"""
    ctm = CTM[ctm] if isinstance(ctm, str) else int(ctm)
    (ih, iw), (oh, ow) = in_hw, out_hw
    compute = scales is None
    if compute:
        hs, ws = F(0), F(0)
    else:
        hs, ws = F(1) / F(scales[0]), F(1) / F(scales[1])
    ho, wo = F(0), F(0)
    ratio = lambda i, o: F(i) / F(o)   # noqa: E731
    corners = lambda i, o: F(0) if o == 1 else F(i - 1) / F(o - 1)   # noqa: E731
    half = lambda s: F(F(0.5) * s) - F(0.5)   # noqa: E731
    if ctm == 0:
        if half_pixel and resize_type != 1:
            if compute:
                hs, ws = ratio(ih, oh), ratio(iw, ow)
            ho, wo = half(hs), half(ws)
        elif align_corners:
            if compute:
                hs, ws = corners(ih, oh), corners(iw, ow)
        elif compute:
            hs, ws = ratio(ih, oh), ratio(iw, ow)
    elif ctm == 1:
        hs, ws = corners(ih, oh), corners(iw, ow)
    elif ctm == 2:
        if compute:
            hs, ws = ratio(ih, oh), ratio(iw, ow)
        ho, wo = half(hs), half(ws)
    elif ctm == 3:
        if oh > 1:
            if compute:
                hs = ratio(ih, oh)
            ho = half(hs)
        elif compute:
            hs = F(0)
        if ow > 1:
            if compute:
                ws = ratio(iw, ow)
            wo = half(ws)
        elif compute:
            ws = F(0)
    elif ctm == 4:
        if compute:
            hs, ws = ratio(ih, oh), ratio(iw, ow)
    elif ctm == 5:
        if compute:
            hs, ws = ratio(ih, oh), ratio(iw, ow)
        ho, wo = F(F(0.5) * hs), F(F(0.5) * ws)
    return ws, hs, wo, ho


def _clamp(v, n):
    return np.clip(v, 0, n - 1).astype(np.int64)


def cubic_weights(t):
    """CubicInterpolation2's four weights at float32 fractions t (array): b float; c float but for a double cubic term; a and d
    double (5.0f * 0.75 is exactly 3.75); each rounded to float32"""
    t = np.asarray(t, F)
    u, ta, td = F(1) - t, F(1) + t, F(2) - t
    d64 = lambda v: np.asarray(v, np.float64)   # noqa: E731
    a = d64(F(3) - F(6) * ta) + 3.75 * d64(ta) * d64(ta) - d64(F(0.75) * ta * ta * ta)
    b = F(1) - F(2.25) * t * t + F(1.25) * t * t * t
    c = d64(F(1) - F(2.25) * u * u) + 1.25 * d64(u) * d64(u) * d64(u)
    d = d64(F(3) - F(6) * td) + 3.75 * d64(td) * d64(td) - d64(F(0.75) * td * td * td)
    return np.stack([a.astype(F), b.astype(F), c.astype(F), d.astype(F)], -1)


def axis_table(resize_type, scale, offset, n_in, n_out):
    """(indices [n_out][taps], weights [n_out][taps] or None) of one axis, in the CPU's float32 expressions"""
    src = np.arange(n_out).astype(F) * F(scale) + F(offset)
    if resize_type == 1:
        return _clamp(np.floor(src), n_in)[:, None], None
    if resize_type == 4:
        return _clamp(np.floor(src + F(0.499)), n_in)[:, None], None
    if resize_type == 2:
        x1 = np.floor(src)
        f = src - x1.astype(F)
        return np.stack([_clamp(x1, n_in), _clamp(x1 + 1, n_in)], -1), np.stack([F(1) - f, f], -1)
    if resize_type == 3:
        x1 = np.trunc(src)
        t = src - np.floor(src)
        return np.stack([_clamp(x1 - 1 + k, n_in) for k in range(4)], -1), cubic_weights(t)
    raise ValueError(f"resize type {resize_type}")


def _weighted(v, w):
    """sum over the last axis of v * w, left to right, each product and sum rounded to float32"""
    s = v[..., 0] * w[..., 0]
    for i in range(1, v.shape[-1]):
        s = s + v[..., i] * w[..., i]
    return s


def interp(x, resize_type, ws, hs, wo, ho, out_hw):
    """y [..., oh, ow] float32 of CPUInterp on x [..., ih, iw] float32 (every leading axis a plane), bit for bit"""
    x = np.asarray(x, F)
    ih, iw = x.shape[-2:]
    oh, ow = out_hw
    xi, xw = axis_table(resize_type, ws, wo, iw, ow)
    yi, yw = axis_table(resize_type, hs, ho, ih, oh)
    if xw is None:
        return x[..., yi[:, 0], :][..., xi[:, 0]]
    rows = x[..., yi, :]                       # [..., oh, taps_y, iw]
    h = _weighted(rows[..., xi], xw)           # [..., oh, taps_y, ow, taps_x] -> [..., oh, taps_y, ow]
    return _weighted(np.moveaxis(h, -2, -1), yw[:, None, :])


def interp64(x, resize_type, ws, hs, wo, ho, out_hw):
    """the same taps and weights applied in float64 (nearest: the same gather)"""
    x = np.asarray(x, np.float64)
    ih, iw = x.shape[-2:]
    oh, ow = out_hw
    xi, xw = axis_table(resize_type, ws, wo, iw, ow)
    yi, yw = axis_table(resize_type, hs, ho, ih, oh)
    if xw is None:
        return x[..., yi[:, 0], :][..., xi[:, 0]]
    h = (x[..., yi, :][..., xi] * xw.astype(np.float64)).sum(-1)
    return (np.moveaxis(h, -2, -1) * yw.astype(np.float64)[:, None, :]).sum(-1)


def out_size(in_hw, out_hw=(0, 0), scale_hw=(0.0, 0.0), scales=None):
    """ShapeInterp's output size: out_hw when both > 0, a scales input (factor * size, truncated), else size * the op's scale"""
    if scales is not None:
        return tuple(int(F(s) * F(i)) for s, i in zip(scales, in_hw))
    if out_hw[0] and out_hw[1]:
        return tuple(out_hw)
    return tuple(int(i * F(s)) for i, s in zip(in_hw, scale_hw))


# ---- the live reference: oracle/_ref/refdump_interp (oracle/refdump_interp.cpp over oracle/_ref/libMNN.so), built by build()
HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(HERE, "_ref")
REFDUMP_INTERP = os.path.join(REF_DIR, "refdump_interp")
DEEPLAB = os.path.join(REF_DIR, "deeplab_f32.mnn")
FPN = os.path.join(REF_DIR, "fpn_f32.mnn")
DEEPLAB_SEED, FPN_SEED = 31, 32


def have_refdump():
    return os.path.exists(REFDUMP_INTERP)


def build_refdump():
    """compile oracle/refdump_interp.cpp against the reference build of oracle/build_ref.py (where the reference sources are) and
    write the DeepLab-v3-style and FPN fixtures with it"""
    from oracle import build_ref as B
    src = os.path.join(HERE, "refdump_interp.cpp")
    lib = os.path.join(REF_DIR, "libMNN.so")
    fresh = have_refdump() and all(os.path.getmtime(REFDUMP_INTERP) > os.path.getmtime(d) for d in (src, lib))
    if not fresh:
        cmd = ["g++", "-O2", "-std=gnu++11", "-w", "-o", REFDUMP_INTERP, src] + ["-I" + os.path.join(B.REF, i) for i in B.INCLUDES] + \
              ["-L" + REF_DIR, "-lMNN", "-Wl,-rpath,$ORIGIN", "-pthread", "-ldl"]
        subprocess.check_call(cmd)
    for path, cmd, seed in ((DEEPLAB, "seg", DEEPLAB_SEED), (FPN, "fpn", FPN_SEED)):
        if not fresh or not os.path.exists(path):
            _run([cmd, path, seed])


def _run(args, plugin=None):
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = REF_DIR + ":" + env.get("LD_LIBRARY_PATH", "")
    env.pop("REFDUMP_PLUGIN", None)
    if plugin:
        env["REFDUMP_PLUGIN"] = plugin
    return subprocess.run([REFDUMP_INTERP] + [str(a) for a in args], env=env, capture_output=True, text=True, timeout=600,
                          check=True)


def ref_interp(x, resize_type, ctm=0, align_corners=False, half_pixel=False, out_hw=(0, 0), scale_hw=(0.0, 0.0), scales=None,
               size_input=None, nhwc=False, x2=None, plugin=None):
    """y (NCHW float32) of one reference Interp op on MNN_FORWARD_CPU.  x NCHW float32; out_hw the op's outputHeight / Width;
    scale_hw its heightScale / widthScale; scales: (h, w) factors of a float scales input [1, 1, h, w]; size_input: (h, w) of an
    int32 size input; nhwc: the input variable is NHWC.  x2: one more input or a list of them, run through the same executor after
    x (all outputs returned, stacked).  plugin: run on MNN_FORWARD_CUDA with that plugin, and (ys, the plugin's stats) returned"""
    x = np.ascontiguousarray(x, F)
    n, c, ih, iw = x.shape
    mode = 1 if scales is not None else (2 if size_input is not None else 0)
    sv = scales if scales is not None else (size_input if size_input is not None else (0, 0))
    hdr = struct.pack("<12i4f", n, c, ih, iw, resize_type, CTM[ctm] if isinstance(ctm, str) else ctm, int(align_corners),
                      int(half_pixel), out_hw[0], out_hw[1], int(nhwc), mode, scale_hw[0], scale_hw[1], float(sv[0]), float(sv[1]))
    more = [] if x2 is None else ([x2] if isinstance(x2, np.ndarray) else list(x2))
    xs = [x] + [np.ascontiguousarray(a, F) for a in more]
    lay = (lambda a: a.transpose(0, 2, 3, 1)) if nhwc else (lambda a: a)   # noqa: E731
    body = b"".join(np.ascontiguousarray(lay(a)).tobytes() for a in xs)
    with tempfile.TemporaryDirectory() as d:
        req, out = os.path.join(d, "req"), os.path.join(d, "out")
        open(req, "wb").write(hdr + struct.pack("<i", len(xs)) + body)
        r = _run(["op", req, out], plugin)
        raw = open(out, "rb").read()
    dims = struct.unpack("<4i", raw[:16])
    ys = np.frombuffer(raw[16:], F).reshape((len(xs),) + dims).copy()
    ys = ys[0] if x2 is None else ys
    if plugin is None:
        return ys
    stats = [json.loads(line) for line in r.stdout.splitlines() if line.startswith('{"plugin_')]
    return ys, (stats[-1] if stats else None)
