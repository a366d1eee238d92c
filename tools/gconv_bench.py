#!/usr/bin/env python3
"""Grouped fp32 convolutions on the split-TF32 wgmma conv kernel (mnnb200_conv_f32_create_grouped), batch 32: one JSON line with,
per layer, the device time (20 executes captured as one CUDA graph, replayed and timed with CUDA events, median of 5 windows),
the algorithmic bytes (input + output + unpacked weights once, fp32) and MACs (M x oc x ic/group x taps) computed from shapes,
the share of the HBM / TF32-over-3 bound reached (the split form issues three TF32 products per MAC), the launch plan, and the same
layer again as a dense group-1 conv with the expanded block-diagonal weights, timed in the same run.  The card's name and power
limit are read in the same call.
Layers: the grouped 3x3 convs of ResNeXt-50 32x4d (all four stages, the stride-2 first blocks included), a RegNet-style layer of
group width 16, a ShuffleNet-v1 g = 3 1x1 and a depth-multiplier-2 3x3 (group = ic, oc = 2 ic).
Usage: python tools/gconv_bench.py [--batch 32] [--iters 20]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BPS, TF32_FLOPS = 3.35e12, 495e12       # H100 SXM data sheet (700 W): the bounds, not reached figures
REPS = 20
# name: ic, oc, group, kernel, stride, input h = w
LAYERS = {
    "resnext_s1_3x3": (128, 128, 32, 3, 1, 56),
    "resnext_s2_first_3x3_s2": (256, 256, 32, 3, 2, 56),
    "resnext_s2_3x3": (256, 256, 32, 3, 1, 28),
    "resnext_s3_first_3x3_s2": (512, 512, 32, 3, 2, 28),
    "resnext_s3_3x3": (512, 512, 32, 3, 1, 14),
    "resnext_s4_first_3x3_s2": (1024, 1024, 32, 3, 2, 14),
    "resnext_s4_3x3": (1024, 1024, 32, 3, 1, 7),
    "regnet_gw16_3x3": (256, 256, 16, 3, 1, 28),
    "shufflenet_g3_1x1": (240, 60, 3, 1, 1, 28),
    "depth_multiplier2_3x3": (32, 64, 32, 3, 1, 56),
}


def time_layer(L, rt, h, x, y, iters):
    import torch
    from mnn_b200 import _capi

    def step():
        for _ in range(REPS):
            _capi.check(L.mnnb200_conv_f32_execute(h, C.c_void_p(x.data_ptr()), C.c_void_p(y.data_ptr())))

    step()
    _capi.check(L.mnnb200_runtime_sync(rt._h))
    g = C.c_void_p()
    _capi.check(L.mnnb200_graph_begin_capture(rt._h))
    step()
    _capi.check(L.mnnb200_graph_end_capture(rt._h, C.byref(g)))
    for _ in range(3):
        L.mnnb200_graph_launch(rt._h, g)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    windows = []
    for _ in range(5):
        e0.record()
        for _ in range(iters):
            L.mnnb200_graph_launch(rt._h, g)
        e1.record()
        torch.cuda.synchronize()
        windows.append(e0.elapsed_time(e1) / (iters * REPS))
    L.mnnb200_graph_destroy(g)
    return sorted(windows)[len(windows) // 2], windows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    import numpy as np
    import torch
    from mnn_b200 import _capi
    from mnn_b200._capi import ConvDesc
    from mnn_b200.backend import Runtime
    if not torch.cuda.is_available():
        sys.exit("gconv_bench: needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True, check=True).stdout.strip().splitlines()[0]
    L = _capi.lib()
    torch.cuda.set_stream(torch.cuda.Stream())
    rt = Runtime(0)
    rng = np.random.default_rng(0)
    n = a.batch
    out = dict(batch=n, card=card, layers={})
    for name, (ic, oc, group, k, s, hw) in LAYERS.items():
        icg, ocg = ic // group, oc // group
        w = (rng.uniform(-1, 1, (oc, icg, k, k)) / np.sqrt(icg * k * k)).astype(np.float32)
        dense = np.zeros((oc, ic, k, k), np.float32)            # block-diagonal: group i's rows see its own input channels
        for g in range(group):
            dense[g * ocg:(g + 1) * ocg, g * icg:(g + 1) * icg] = w[g * ocg:(g + 1) * ocg]
        x = torch.randn(n, ic, hw, hw, device="cuda")
        row = {}
        for form, weights, grp in (("grouped", w, group), ("dense", dense, 1)):
            d = ConvDesc(ic, oc, k, k, s, s, k // 2, k // 2, 1, 1, grp, 0)
            h = C.c_void_p()
            f = L.mnnb200_conv_f32_create_grouped if grp > 1 else L.mnnb200_conv_f32_create
            _capi.check(f(rt._h, C.byref(d), weights.ctypes.data_as(C.c_void_p), None, 0, C.byref(h)))
            try:
                oh, ow = C.c_int(0), C.c_int(0)
                _capi.check(L.mnnb200_conv_f32_resize(h, n, hw, hw, C.byref(oh), C.byref(ow)))
                y = torch.empty(n, oc, oh.value, ow.value, device="cuda")
                fields = (C.c_int * 9)()
                _capi.check(L.mnnb200_conv_f32_plan(h, fields, 9))
                ms, windows = time_layer(L, rt, h, x, y, a.iters)
            finally:
                L.mnnb200_exec_destroy(h)
            macs = n * oh.value * ow.value * oc * icg * k * k         # the grouped conv's work, for both forms
            bytes_ = 4.0 * (n * ic * hw * hw + n * oc * oh.value * ow.value + oc * icg * k * k)
            bound_ms = max(bytes_ / HBM_BPS, 3 * 2 * macs / TF32_FLOPS) * 1e3
            row[form] = dict(device_ms=round(ms, 4), ms_windows=[round(v, 4) for v in windows],
                             plan=dict(zip(("bn", "n_chunks", "m_tiles", "num_kb", "stages", "cp8", "taps", "P", "Q"), fields)),
                             algorithmic_bytes=bytes_, macs=macs, GBps=round(bytes_ / ms / 1e6, 1),
                             bound="hbm" if bytes_ / HBM_BPS > 6 * macs / TF32_FLOPS else "tf32/3",
                             bound_ms=round(bound_ms, 4), share_of_bound=round(bound_ms / ms, 3))
        row["shape"] = dict(ic=ic, oc=oc, group=group, kernel=k, stride=s, hw=hw)
        row["dense_over_grouped"] = round(row["dense"]["device_ms"] / row["grouped"]["device_ms"], 2)
        out["layers"][name] = row
    out["grouped_total_ms"] = round(sum(r["grouped"]["device_ms"] for r in out["layers"].values()), 4)
    out["dense_total_ms"] = round(sum(r["dense"]["device_ms"] for r in out["layers"].values()), 4)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
