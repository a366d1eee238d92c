"""Float64 restatement of the reference CPU's fp32 Deconvolution (CPUDeconvolution, CPUDeconvolutionDepthwise), in its scatter
form: every input pixel adds x[n][ic][iy][ix] * w[ic][oc][ky][kx] to output (iy * sh - pad_t + ky * dh, ix * sw - pad_l + kx * dw)
when that lies inside the output; then + bias, then ReLU / ReLU6 (CPUDeconvolution.cpp, the GEMM into a column buffer and the
col2im scatter-add with dilation, then the post parameters)."""
import json
import os
import struct
import subprocess
import tempfile

import numpy as np


def pair(v):
    return tuple(v) if isinstance(v, (tuple, list)) else (v, v)


def natural_out(i, k, s, p, d):
    """ShapeDeconvolution.cpp with symmetric pads and no out-pad: (i - 1) * s + d * (k - 1) + 1 - 2 * p"""
    return (i - 1) * s + d * (k - 1) + 1 - 2 * p


def deconv_f32(x, w, b, stride=1, pad=0, dil=1, act=0, out_hw=None, depthwise=False):
    """(y, S) in float64.  x [n][ic][ih][iw]; w [ic][oc][kh][kw], or [c][kh][kw] / [c][1][kh][kw] when depthwise; b [oc] or None;
    pad = the begin pads (top, left) from ConvolutionCommon::convolutionTransposePad; out_hw the output size (natural when None);
    act 0 none, 1 ReLU, 2 ReLU6.  S = deconv(|x|, |w|) over the same taps, no bias: the magnitude sum error bounds scale with."""
    x = np.asarray(x, np.float64)
    w = np.asarray(w, np.float64)
    if depthwise:
        w = w.reshape(w.shape[0], w.shape[-2], w.shape[-1])
    n, ic, ih, iw = x.shape
    oc = ic if depthwise else w.shape[1]
    kh, kw = w.shape[-2:]
    (sh, sw), (pt, pl), (dh, dw) = pair(stride), pair(pad), pair(dil)
    oh, ow = out_hw or (natural_out(ih, kh, sh, pt, dh), natural_out(iw, kw, sw, pl, dw))
    fh, fw = max((ih - 1) * sh + dh * (kh - 1) + 1, pt + oh), max((iw - 1) * sw + dw * (kw - 1) + 1, pl + ow)

    def scatter(xx, ww):
        full = np.zeros((n, oc, fh, fw))
        for ky in range(kh):
            for kx in range(kw):
                if depthwise:
                    t = xx * ww[None, :, ky, kx, None, None]
                else:
                    t = np.einsum("nihw,io->nohw", xx, ww[:, :, ky, kx])
                full[:, :, ky * dh:ky * dh + (ih - 1) * sh + 1:sh, kx * dw:kx * dw + (iw - 1) * sw + 1:sw] += t
        return full[:, :, pt:pt + oh, pl:pl + ow]

    y = scatter(x, w)
    if b is not None:
        y = y + np.asarray(b, np.float64)[None, :, None, None]
    if act >= 1:
        y = np.maximum(y, 0)
    if act == 2:
        y = np.minimum(y, 6)
    return y, scatter(np.abs(x), np.abs(w))


# ---- the live reference: oracle/_ref/refdump_deconv (oracle/refdump_deconv.cpp over oracle/_ref/libMNN.so), built by build()
HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(HERE, "_ref")
REFDUMP_DECONV = os.path.join(REF_DIR, "refdump_deconv")


def have_refdump():
    return os.path.exists(REFDUMP_DECONV)


def build_refdump():
    """compile oracle/refdump_deconv.cpp against the reference build of oracle/build_ref.py (where the reference sources are)"""
    from oracle import build_ref as B
    src = os.path.join(HERE, "refdump_deconv.cpp")
    lib = os.path.join(REF_DIR, "libMNN.so")
    if have_refdump() and all(os.path.getmtime(REFDUMP_DECONV) > os.path.getmtime(d) for d in (src, lib)):
        return
    cmd = ["g++", "-O2", "-std=gnu++11", "-w", "-o", REFDUMP_DECONV, src] + ["-I" + os.path.join(B.REF, i) for i in B.INCLUDES] + \
          ["-L" + REF_DIR, "-lMNN", "-Wl,-rpath,$ORIGIN", "-pthread", "-ldl"]
    subprocess.check_call(cmd)


def _run(args, plugin=None):
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = REF_DIR + ":" + env.get("LD_LIBRARY_PATH", "")
    env.pop("REFDUMP_PLUGIN", None)
    if plugin:
        env["REFDUMP_PLUGIN"] = plugin
    return subprocess.run([REFDUMP_DECONV] + [str(a) for a in args], env=env, capture_output=True, text=True, timeout=600,
                          check=True)


def ref_deconv(x, w, b, stride=1, pads=(0, 0, 0, 0), dil=1, out_pads=(0, 0), same=False, out_hw=None, depthwise=False, relu=False,
               relu6=False, plugin=None):
    """y of the reference's Deconvolution on MNN_FORWARD_CPU; pads [t, l, b, r].  plugin: the plugin library, run on
    MNN_FORWARD_CUDA, and (y, the plugin's {plugin_created, plugin_declined}) returned"""
    x = np.ascontiguousarray(x, np.float32)
    w = np.ascontiguousarray(w, np.float32)
    n, ic, ih, iw = x.shape
    oc = ic if depthwise else w.shape[1]
    kh, kw = w.shape[-2:]
    (sh, sw), (dh, dw) = pair(stride), pair(dil)
    oh, ow = out_hw or (0, 0)
    hdr = struct.pack("<24i", n, ic, ih, iw, oc, kh, kw, sh, sw, *pads, dh, dw, *out_pads, int(same), oh, ow, int(depthwise),
                      int(relu), int(relu6), int(b is not None))
    body = x.tobytes() + w.tobytes() + (np.ascontiguousarray(b, np.float32).tobytes() if b is not None else b"")
    with tempfile.TemporaryDirectory() as d:
        req, out = os.path.join(d, "req"), os.path.join(d, "out")
        open(req, "wb").write(hdr + body)
        r = _run(["deconv", req, out], plugin)
        raw = open(out, "rb").read()
    dims = struct.unpack("<4i", raw[:16])
    y = np.frombuffer(raw[16:], np.float32).reshape(dims).copy()
    if plugin is None:
        return y
    stats = [json.loads(line) for line in r.stdout.splitlines() if line.startswith('{"plugin_')]
    return y, (stats[-1] if stats else None)


def ref_chain(batch, seed, plugin=None):
    """conv 3x3 -> deconv 4x4 s2 -> depthwise deconv 3x3 -> conv 1x1 run twice, with two inputs, on one executor (refdump_deconv
    chain): ({name_run: fp32 array} for the deconvolution's and the graph's outputs, the plugin's stats or None)"""
    with tempfile.TemporaryDirectory() as d:
        r = _run(["chain", batch, seed, d], plugin)
        out = {f[:-4]: np.fromfile(os.path.join(d, f), np.float32) for f in os.listdir(d)}
    stats = [json.loads(line) for line in r.stdout.splitlines() if line.startswith('{"plugin_')]
    return out, (stats[-1] if stats else None)
