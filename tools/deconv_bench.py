#!/usr/bin/env python3
"""fp32 Deconvolution at sizes users run, one JSON line per layer, each with:
  ms            device time per launch of mnnb200_deconv_f32_execute (CUDA events around --iters back-to-back launches, after
                --warmup), the split-TF32 phase-decomposed kernel;
  bytes, flops  algorithmic bytes (input + output + weights once, fp32) and FLOPs (2 x MACs of the transposed conv; the split form
                issues 3x that on the tensor cores), from shapes;
  bound         the share of the limiting bound reached: HBM 3.35 TB/s, or TF32 495 TFLOP/s / 3 for the split (H100 SXM data
                sheet at 700 W; the bounds, not reached figures), and which one limits;
  zero_insert_ms  in the same run, the naive alternative: the input scattered into a zero-filled buffer with stride-sized gaps,
                then the existing fp32 conv kernel (mnnb200_conv_f32_execute, flipped and transposed weights, stride 1) on it, both
                timed together;
  card          name and power limit, read in the same call.
Usage: python tools/deconv_bench.py [--iters 50] [--warmup 10]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BPS, TF32_SPLIT_FLOPS = 3.35e12, 495e12 / 3
# name: batch, ic, oc, (ih, iw), kernel, stride, pad
LAYERS = [
    ("simplebaseline_head_1", 32, 2048, 256, (8, 6), 4, 2, 1),
    ("simplebaseline_head_2", 32, 256, 256, (16, 12), 4, 2, 1),
    ("simplebaseline_head_3", 32, 256, 256, (32, 24), 4, 2, 1),
    ("unet_up_512_256", 8, 512, 256, (28, 28), 2, 2, 0),
    ("unet_up_256_128", 8, 256, 128, (56, 56), 2, 2, 0),
    ("fcn8s_up8", 8, 21, 21, (28, 28), 16, 8, 4),
]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        return q
    except (OSError, subprocess.CalledProcessError, IndexError):
        return "unknown"


def timed(fn, iters, warmup):
    import torch
    for _ in range(warmup):
        fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    import numpy as np
    import torch
    assert torch.cuda.is_available(), "deconv_bench times the GPU: no CUDA device"
    from mnn_b200 import _capi
    from mnn_b200._capi import ConvDesc
    from mnn_b200.backend import Runtime
    L, D = _capi.lib(), _capi.deconv_lib()
    torch.cuda.set_stream(torch.cuda.Stream())   # the runtime adopts torch's current stream: fills, copies and kernels in order
    rt = Runtime(0)
    dev_card = card()
    rng = np.random.default_rng(0)
    for name, n, ic, oc, (ih, iw), k, s, p in LAYERS:
        w = (rng.uniform(-1, 1, (ic, oc, k, k)) / np.sqrt(ic * k * k)).astype(np.float32)
        h = C.c_void_p()
        d = ConvDesc(ic, oc, k, k, s, s, p, p, 1, 1, 1, 0)
        _capi.check(D.mnnb200_deconv_f32_create(rt._h, C.byref(d), w.ctypes.data_as(C.c_void_p), None, 0, C.byref(h)))
        oh, ow = C.c_int(0), C.c_int(0)
        _capi.check(D.mnnb200_deconv_f32_resize(h, n, ih, iw, C.byref(oh), C.byref(ow)))
        oh, ow = oh.value, ow.value
        x = torch.randn((n, ic, ih, iw), device="cuda")
        y = torch.empty((n, oc, oh, ow), device="cuda")
        ms = timed(lambda: _capi.check(D.mnnb200_deconv_f32_execute(h, C.c_void_p(x.data_ptr()), C.c_void_p(y.data_ptr()))),
                   a.iters, a.warmup)
        # the zero-insert baseline: x at stride s in a zero buffer padded by k - 1 - p, then a stride-1 conv with the flipped,
        # transposed kernel gives the same output
        e = k - 1 - p
        zh, zw = (ih - 1) * s + 1 + 2 * e, (iw - 1) * s + 1 + 2 * e
        z = torch.zeros((n, ic, zh, zw), device="cuda")
        wc = np.ascontiguousarray(w.transpose(1, 0, 2, 3)[:, :, ::-1, ::-1])
        hc = C.c_void_p()
        dc = ConvDesc(ic, oc, k, k, 1, 1, 0, 0, 1, 1, 1, 0)
        _capi.check(L.mnnb200_conv_f32_create(rt._h, C.byref(dc), wc.ctypes.data_as(C.c_void_p), None, 0, C.byref(hc)))
        ch, cw = C.c_int(oh), C.c_int(ow)
        _capi.check(L.mnnb200_conv_f32_resize(hc, n, zh, zw, C.byref(ch), C.byref(cw)))
        yz = torch.empty((n, oc, oh, ow), device="cuda")
        view = z[:, :, e:e + (ih - 1) * s + 1:s, e:e + (iw - 1) * s + 1:s]

        def naive():
            view.copy_(x)
            _capi.check(L.mnnb200_conv_f32_execute(hc, C.c_void_p(z.data_ptr()), C.c_void_p(yz.data_ptr())))

        zms = timed(naive, a.iters, a.warmup)
        torch.cuda.synchronize()
        agree = float((y - yz).abs().max() / y.abs().max())
        nbytes = 4.0 * (n * ic * ih * iw + n * oc * oh * ow + ic * oc * k * k)
        flops = 2.0 * n * ih * iw * ic * oc * k * k
        t_hbm, t_mma = nbytes / HBM_BPS, flops / TF32_SPLIT_FLOPS
        print(json.dumps(dict(layer=name, batch=n, ic=ic, oc=oc, input=[ih, iw], output=[oh, ow], kernel=k, stride=s, pad=p,
                              ms=round(ms, 4), bytes=nbytes, flops=flops, bound="tf32_split" if t_mma > t_hbm else "hbm",
                              share_of_bound=round(max(t_hbm, t_mma) * 1e3 / ms, 3), zero_insert_ms=round(zms, 4),
                              speedup_vs_zero_insert=round(zms / ms, 2), max_rel_diff_vs_zero_insert=agree, card=dev_card)),
              flush=True)
        L.mnnb200_exec_destroy(h)
        L.mnnb200_exec_destroy(hc)


if __name__ == "__main__":
    main()
