"""fp32 GridSample (mnnb200_grid_sample_f32_*) at shapes users run: a 1/4-resolution flow warp (32 x 64 x 64^2, equal in and out),
a full-resolution RGB warp (8 x 3 x 512^2), deformable-style sampling (8 x 256 x 64^2 -> 32^2), a 3D-LUT lookup (8 x 3 x 33^3 ->
512^2) and a nearest 5-D resampling.  One JSON line per shape: device us per launch (CUDA events over back-to-back launches after
a warm-up, best of 5 rounds, and the spread), bytes (output written once, grid read once, input read once) and their share of the
3.35 TB/s HBM bound, torch.nn.functional.grid_sample on the same tensors alternating in the same process (speed; for bilinear
zeros / border also its max relative difference at the timed size), the plan, card name and power limit.
Run: python tools/grid_sample_bench.py [--iters 50]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM = 3.35e12
PLAN_FIELDS = ("rank", "taps", "cgroups", "cper", "grid", "threads", "vec")
# name: (x shape, grid spatial dims, mode, padding, align_corners)
SHAPES = {
    "flow_warp_quarter_res": ((32, 64, 64, 64), (64, 64), "bilinear", "zeros", False),
    "rgb_warp_full_res": ((8, 3, 512, 512), (512, 512), "bilinear", "border", False),
    "deformable_256ch_64_to_32": ((8, 256, 64, 64), (32, 32), "bilinear", "zeros", False),
    "lut3d_33_to_512": ((8, 3, 33, 33, 33), (1, 512, 512), "bilinear", "border", True),
    "nearest_5d_16ch_32": ((4, 16, 32, 32, 32), (32, 32, 32), "nearest", "zeros", False),
}
MODE, PAD = {"bilinear": 0, "nearest": 1}, {"zeros": 0, "border": 1}


def timed(fn, iters, rounds=5):
    """best and spread of `rounds` windows of `iters` back-to-back launches, us per launch (events on torch's default stream, which
    the runtime adopts)"""
    import torch
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    res = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        res.append(a.elapsed_time(b) * 1e3 / iters)
    return min(res), max(res) - min(res)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    import torch
    from mnn_b200 import _capi
    from mnn_b200.backend import Runtime
    backend = Runtime(0).onCreate()
    L, GS = _capi.lib(), _capi.grid_sample_lib()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                          check=True).stdout.strip().splitlines()[0]
    gen = torch.Generator(device="cuda").manual_seed(0)
    for name, (xs, outd, mode, pad, align) in SHAPES.items():
        rank = len(xs)
        x = torch.randn(xs, device="cuda", generator=gen)
        g = torch.rand((xs[0],) + outd + (rank - 2,), device="cuda", generator=gen) * 2.2 - 1.1
        y = torch.empty((xs[0], xs[1]) + outd, device="cuda")
        h = C.c_void_p()
        assert GS.mnnb200_grid_sample_f32_create(backend.runtime._h, MODE[mode], PAD[pad], int(align), C.byref(h)) == 0
        ind, od = (C.c_int * (rank - 2))(*xs[2:]), (C.c_int * (rank - 2))(*outd)
        assert GS.mnnb200_grid_sample_f32_resize(h, rank, xs[0], xs[1], ind, od) == 0, L.mnnb200_last_error()

        def ours():
            GS.mnnb200_grid_sample_f32_execute(h, C.c_void_p(x.data_ptr()), C.c_void_p(g.data_ptr()), C.c_void_p(y.data_ptr()))

        def theirs():
            return torch.nn.functional.grid_sample(x, g, mode=mode, padding_mode=pad, align_corners=align)
        us, spread, tus, tspread = [], [], [], []
        for _ in range(2):   # alternate: ours, torch, ours, torch
            m, s = timed(ours, a.iters)
            us.append(m); spread.append(s)
            m, s = timed(theirs, a.iters)
            tus.append(m); tspread.append(s)
        torch.cuda.synchronize()
        backend.onSync()
        f = (C.c_int * len(PLAN_FIELDS))()
        assert GS.mnnb200_grid_sample_f32_plan(h, f, len(PLAN_FIELDS)) == 0
        L.mnnb200_exec_destroy(h)
        nbytes = 4 * (y.numel() + g.numel() + x.numel())
        best, tbest = min(us), min(tus)
        res = dict(shape=name, x=list(xs), out=list(outd), mode=mode, padding=pad, align_corners=align, us_per_launch=round(best, 2),
                   spread_us=round(max(spread), 2), bytes=nbytes, hbm_share=round(nbytes / HBM / (best * 1e-6), 3),
                   torch_us=round(tbest, 2), torch_spread_us=round(max(tspread), 2), speedup_vs_torch=round(tbest / best, 2),
                   plan=dict(zip(PLAN_FIELDS, f)), card=card)
        if mode == "bilinear":
            ref = theirs()
            res["torch_max_rel_diff"] = float((y - ref).abs().max() / ref.abs().max().clamp_min(1e-12))
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
