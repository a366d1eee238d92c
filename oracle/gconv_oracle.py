"""Float64 restatement of the reference CPU's grouped fp32 Convolution (ConvolutionFloatFactory + ConvolutionGroup): group i is an
ordinary convolution over input channels [i icg, (i+1) icg) with weights w[i ocg:(i+1) ocg] ([oc][icg][kh][kw]) and bias
b[i ocg:(i+1) ocg]; then ReLU / ReLU6.  The group is common->group(), unless inputCount > 0 differs from the input's channel count,
when it is channels / inputCount (`cpu_group`)."""
import json
import os
import struct
import subprocess
import tempfile

import numpy as np


def pair(v):
    return tuple(v) if isinstance(v, (tuple, list)) else (v, v)


def cpu_group(group, input_count, channels):
    """ConvolutionFloatFactory.cpp: the group the CPU splits the conv into"""
    return channels // input_count if 0 < input_count != channels else group


def out_size(i, k, s, p0, p1, d):
    return (i + p0 + p1 - d * (k - 1) - 1) // s + 1


def gconv_f32(x, w, b, group, stride=1, pads=(0, 0, 0, 0), dil=1, act=0):
    """(y, S) in float64.  x [n][ic][ih][iw]; w [oc][ic / group][kh][kw]; b [oc] or None; pads [t, l, b, r]; act 0 none, 1 ReLU,
    2 ReLU6.  S = the same conv of |x| and |w| with no bias: the magnitude sum error bounds scale with."""
    import torch
    import torch.nn.functional as F
    x = torch.from_numpy(np.asarray(x, np.float64))
    w = torch.from_numpy(np.asarray(w, np.float64))
    oc, icg, kh, kw = w.shape
    assert x.shape[1] == icg * group and oc % group == 0, (x.shape, w.shape, group)
    pt, pl, pb, pr = pads
    xp = F.pad(x, (pl, pr, pt, pb))

    def conv(xx, ww):
        return F.conv2d(xx, ww, None, pair(stride), 0, pair(dil), group)

    y = conv(xp, w)
    if b is not None:
        y = y + torch.from_numpy(np.asarray(b, np.float64))[None, :, None, None]
    if act >= 1:
        y = y.clamp(min=0)
    if act == 2:
        y = y.clamp(max=6)
    return y.numpy(), conv(xp.abs(), w.abs()).numpy()


# ---- the live reference: oracle/_ref/refdump_gconv (oracle/refdump_gconv.cpp over oracle/_ref/libMNN.so), built by build()
HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(HERE, "_ref")
REFDUMP_GCONV = os.path.join(REF_DIR, "refdump_gconv")
RESNEXT = os.path.join(REF_DIR, "resnext50_f32.mnn")
RESNEXT_SEED = 29


def have_refdump():
    return os.path.exists(REFDUMP_GCONV)


def build_refdump():
    """compile oracle/refdump_gconv.cpp against the reference build of oracle/build_ref.py (where the reference sources are) and
    write the ResNeXt-50 fixture with it"""
    from oracle import build_ref as B
    src = os.path.join(HERE, "refdump_gconv.cpp")
    lib = os.path.join(REF_DIR, "libMNN.so")
    fresh = have_refdump() and all(os.path.getmtime(REFDUMP_GCONV) > os.path.getmtime(d) for d in (src, lib))
    if not fresh:
        cmd = ["g++", "-O2", "-std=gnu++11", "-w", "-o", REFDUMP_GCONV, src] + \
              ["-I" + os.path.join(B.REF, i) for i in B.INCLUDES] + ["-L" + REF_DIR, "-lMNN", "-Wl,-rpath,$ORIGIN", "-pthread", "-ldl"]
        subprocess.check_call(cmd)
    if not fresh or not os.path.exists(RESNEXT):
        _run(["resnext", RESNEXT, RESNEXT_SEED])


def _run(args, plugin=None):
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = REF_DIR + ":" + env.get("LD_LIBRARY_PATH", "")
    env.pop("REFDUMP_PLUGIN", None)
    if plugin:
        env["REFDUMP_PLUGIN"] = plugin
    return subprocess.run([REFDUMP_GCONV] + [str(a) for a in args], env=env, capture_output=True, text=True, timeout=600,
                          check=True)


def _stats(r):
    stats = [json.loads(line) for line in r.stdout.splitlines() if line.startswith('{"plugin_')]
    return stats[-1] if stats else None


def ref_gconv(x, w, b, group, input_count=0, stride=1, pads=(0, 0, 0, 0), dil=1, relu=False, relu6=False, plugin=None):
    """y of the reference's Convolution (common->group = group, inputCount = input_count) on MNN_FORWARD_CPU; w holds
    oc * (ic / cpu_group) * kh * kw values.  plugin: the plugin library, run on MNN_FORWARD_CUDA, and (y, the plugin's
    {plugin_created, plugin_declined}) returned"""
    x = np.ascontiguousarray(x, np.float32)
    w = np.ascontiguousarray(w, np.float32)
    n, ic, ih, iw = x.shape
    oc, _, kh, kw = w.shape
    (sh, sw), (dh, dw) = pair(stride), pair(dil)
    hdr = struct.pack("<21i", n, ic, ih, iw, oc, kh, kw, sh, sw, *pads, dh, dw, group, input_count, int(relu), int(relu6),
                      int(b is not None), w.size)
    body = x.tobytes() + w.tobytes() + (np.ascontiguousarray(b, np.float32).tobytes() if b is not None else b"")
    with tempfile.TemporaryDirectory() as d:
        req, out = os.path.join(d, "req"), os.path.join(d, "out")
        open(req, "wb").write(hdr + body)
        r = _run(["conv", req, out], plugin)
        raw = open(out, "rb").read()
    dims = struct.unpack("<4i", raw[:16])
    y = np.frombuffer(raw[16:], np.float32).reshape(dims).copy()
    return y if plugin is None else (y, _stats(r))


def ref_block(batch, seed, plugin=None):
    """two ResNeXt bottlenecks run twice, with two inputs, on one executor (refdump_gconv block): ({name_run: fp32 array} for the
    first block's grouped conv and the graph's output, the plugin's stats or None)"""
    with tempfile.TemporaryDirectory() as d:
        r = _run(["block", batch, seed, d], plugin)
        out = {f[:-4]: np.fromfile(os.path.join(d, f), np.float32) for f in os.listdir(d)}
    return out, _stats(r)
