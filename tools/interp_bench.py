#!/usr/bin/env python3
"""fp32 Interp at sizes users run, one JSON line per shape, each with:
  us            device time per launch of mnnb200_interp_f32_execute (CUDA events around --iters back-to-back launches, after
                --warmup);
  bytes         the input read once and the output written once (fp32), from shapes;
  hbm_share     the share of the HBM bound that is: bytes / 3.35 TB/s (H100 SXM data sheet at 700 W; the bound, not a reached
                figure) over the measured time;
  torch_us      in the same process, alternating with the kernel, torch.nn.functional.interpolate on the same tensors with the
                nearest mode or the bilinear / bicubic mode and align_corners of the shape: a yardstick for speed only, its
                arithmetic differs from MNN's;
  card          name and power limit, read in the same call.
Usage: python tools/interp_bench.py [--iters 200] [--warmup 20] [--rounds 5]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BPS = 3.35e12
# name: n, c, (ih, iw), (oh, ow), resize type, ctm
SHAPES = [
    ("deeplab_decoder_x4_align", 8, 256, (64, 64), (256, 256), 2, "AlignCorners"),
    ("logits_x8_bilinear", 8, 21, (64, 64), (512, 512), 2, "PytorchHalfPixels"),
    ("image_pool_1x1_to_64", 8, 256, (1, 1), (64, 64), 2, "PytorchHalfPixels"),
    ("fpn_20_to_40_nearest", 16, 256, (20, 20), (40, 40), 1, "NotSet"),
    ("fpn_40_to_80_nearest", 16, 128, (40, 40), (80, 80), 1, "NotSet"),
    ("down_half_bilinear", 8, 64, (256, 256), (128, 128), 2, "HalfPixels"),
    ("cubic_256_to_512", 8, 3, (256, 256), (512, 512), 3, "PytorchHalfPixels"),
]
TORCH_MODE = {1: "nearest", 2: "bilinear", 3: "bicubic", 4: "nearest"}


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError, IndexError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    import torch
    import torch.nn.functional as Fn
    assert torch.cuda.is_available(), "interp_bench needs an H100 (there is no CPU path)"
    from mnn_b200 import _capi
    from mnn_b200.backend import Runtime
    from oracle import interp_oracle as I
    rt = Runtime(0).onCreate().runtime
    L = _capi.interp_lib()
    who = card()
    print(json.dumps({"card": who}))
    for name, n, c, ihw, ohw, rtype, ctm in SHAPES:
        x = torch.randn(n, c, *ihw, device="cuda")
        y = torch.empty(n, c, *ohw, device="cuda")
        ws, hs, wo, ho = (float(v) for v in I.transform(rtype, ctm, 0, 0, ihw, ohw))
        h = C.c_void_p()
        _capi.check(L.mnnb200_interp_f32_create(rt._h, rtype, ws, hs, wo, ho, C.byref(h)), "interp_f32_create")
        _capi.check(L.mnnb200_interp_f32_resize(h, n * c, ihw[0], ihw[1], ohw[0], ohw[1]), "interp_f32_resize")
        xp, yp = C.c_void_p(x.data_ptr()), C.c_void_p(y.data_ptr())
        kw = {} if rtype in (1, 4) else {"align_corners": ctm == "AlignCorners"}

        def ours():
            L.mnnb200_interp_f32_execute(h, xp, yp)

        def theirs():
            Fn.interpolate(x, size=ohw, mode=TORCH_MODE[rtype], **kw)

        def timed(fn):
            for _ in range(a.warmup):
                fn()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(a.iters):
                fn()
            e.record()
            e.synchronize()
            return s.elapsed_time(e) * 1e3 / a.iters

        t_ours, t_torch = [], []
        for _ in range(a.rounds):
            t_ours.append(timed(ours))
            t_torch.append(timed(theirs))
        f = (C.c_int * 7)()
        _capi.check(L.mnnb200_interp_f32_plan(h, f, 7), "interp_f32_plan")
        _capi.lib().mnnb200_exec_destroy(h)
        nbytes = 4 * n * c * (ihw[0] * ihw[1] + ohw[0] * ohw[1])
        us = min(t_ours)
        print(json.dumps({"shape": name, "n": n, "c": c, "in": ihw, "out": ohw, "resize_type": rtype, "ctm": ctm,
                          "us": round(us, 2), "us_spread": [round(min(t_ours), 2), round(max(t_ours), 2)], "bytes": nbytes,
                          "hbm_share": round(nbytes / HBM_BPS / (us * 1e-6), 3), "torch_us": round(min(t_torch), 2),
                          "vec": f[1], "grid": f[2], "card": who}))


if __name__ == "__main__":
    main()
