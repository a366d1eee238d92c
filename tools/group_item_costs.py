"""Cost of one work item of the persistent conv-group launch (conv_group_wgmma.cu), per CTA: single-layer groups of a 1x1 int8
conv at M = 32 x 112 x 112 rows (about 24 items of 128 rows per CTA on a 132-SM part), swept over the tile width (OC at
K = 16) and over K (at OC = 32), plus the shallow 1x1 shapes of MobileNet-v2's first blocks.  Each configuration is one group launch captured in a CUDA graph and replayed back to back;
the time is the median of several windows.  "kernel" is the launch the plan chose for the layer: the conv-group kernel
(128-row items on two consumer warpgroups) or, for one-K-block layers up to 96 wide, the shallow kernel (the same 128-row items
split into 64-row halves over four consumer warpgroups).  Cycles use the SM clock read while the replays run.  Next to each: the
algorithmic bytes (input + output activations, weights) and the time they take at the data-sheet HBM bandwidth.
Usage (on the GPU): python tools/group_item_costs.py > item_costs.json"""
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from mnn_b200 import _capi  # noqa: E402
from mnn_b200.backend import ConvGroupExecution, Op, QuantAttr, Runtime, Tensor  # noqa: E402

PEAK_GBS = 3350.0     # H100 SXM data-sheet HBM3 bandwidth
N, H, W = 32, 112, 112
SWEEP_OC = [(16, oc) for oc in (16, 32, 64, 96, 128)]          # (K, OC)
SWEEP_K = [(k, 32) for k in (16, 64, 128, 256, 576)]
SHALLOW = [(16, 16), (32, 16), (16, 96), (32, 144)]


def smi(query):
    out = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i",
                          str(torch.cuda.current_device())], capture_output=True, text=True, check=True).stdout
    return out.strip().splitlines()[0]


def up16(c):
    return (c + 15) // 16 * 16


def measure(backend, stream, k, oc, steps=100, reps=7):
    rng = np.random.default_rng(k * 1000 + oc)
    w = rng.integers(-127, 128, (oc, k, 1, 1)).astype(np.int8)
    ws = (rng.uniform(0.002, 0.02, oc) / np.sqrt(k)).astype(np.float32)
    bias = rng.uniform(-1, 1, oc).astype(np.float32)
    op = Op(type="ConvInt8", conv=dict(ic=k, oc=oc, kernel=(1, 1), stride=(1, 1), pad=(0, 0), relu=True),
            weight=w, wscale=ws, bias=bias)
    qi, qo = QuantAttr(0.05, 2, -128, 127), QuantAttr(0.07, -3, -127, 127)
    xin = backend.onAcquire(Tensor((N, k, H, W), "int8", qi))
    xin.data.copy_(torch.randint(-128, 128, xin.data.shape, dtype=torch.int8))
    yout = Tensor((N, oc, 1, 1), "int8", qo)
    ex = backend.onCreate([xin], [yout], op)
    assert ex.onResize([xin], [yout]) == 0
    backend.onAcquire(yout)
    assert ConvGroupExecution.groupable(ex)
    grp = ConvGroupExecution(backend, [ex])
    assert grp.bind([xin], [yout]) == 0
    with torch.cuda.stream(stream):
        assert grp.onExecute() == 0
    stream.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        assert grp.onExecute() == 0
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(stream):
        for _ in range(20):
            g.replay()
    stream.synchronize()
    times, clocks = [], []
    for _ in range(reps):
        with torch.cuda.stream(stream):
            ev0.record()
            for _ in range(steps):
                g.replay()
            ev1.record()
        clocks.append(float(smi("clocks.sm")))           # read while the window's replays are still running
        stream.synchronize()
        times.append(ev0.elapsed_time(ev1) * 1e3 / steps)
    f = (C.c_int * 11)()
    assert _capi.lib().mnnb200_conv_int8_group_plan(ex._h, f, 11) == 0
    us = sorted(times)[len(times) // 2]
    mhz = sorted(clocks)[len(clocks) // 2]
    M = N * H * W
    items = (M + 127) // 128 * -(-up16(oc) // min(up16(oc), 128))
    grid = min(items, backend.runtime.sm_count)
    per_cta = items / grid
    alg = M * up16(k) + M * up16(oc) + up16(oc) * up16(k)
    return {"K": k, "OC": oc, "kernel": ("conv_group", "shallow")[f[10]], "us": round(us, 2), "items": items, "items_per_cta": round(per_cta, 2),
            "us_per_item": round(us / per_cta, 3), "cycles_per_item": round(us / per_cta * mhz),
            "sm_mhz": mhz, "alg_MB": round(alg / 1e6, 2), "hbm_us": round(alg / PEAK_GBS / 1e3, 2),
            "share_of_hbm": round(alg / PEAK_GBS / 1e3 / us, 3)}


def main():
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        backend = Runtime(torch.cuda.current_device()).onCreate()
    rows = {"oc_at_k16": [measure(backend, stream, k, oc) for k, oc in SWEEP_OC],
            "k_at_oc32": [measure(backend, stream, k, oc) for k, oc in SWEEP_K],
            "shallow_1x1": [measure(backend, stream, k, oc) for k, oc in SHALLOW]}
    print(json.dumps({"device": torch.cuda.get_device_name(), "power_limit_w": smi("power.limit"),
                      "sm_count": backend.runtime.sm_count, "M": N * H * W, **rows}, indent=1))


if __name__ == "__main__":
    main()
