"""LSTM / RNN through the C ABI (mnnb200_rnn_*) at sizes users run, against torch.nn.LSTM / nn.RNN in fp32 on cuDNN (TF32 off)
in the same process: a CRNN recogniser's two bidirectional layers (T 32, B 32, I 256 -> H 256), streaming speech (T 200, B 16,
I 80 -> H 512), a keyword-spotting chunk with states (T 16, B 1, I 40 -> H 128) and a streamed-R layer (T 100, B 64, H 1024).
One JSON line per case: device µs per execute (CUDA events over back-to-back executes, best of 5 rounds), µs per step, the
projection MatMul and the recurrence timed apart (the MatMul alone through mnnb200_matmul_*), cuDNN's µs, the plan, card name
and power limit."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CASES = {  # name: (cell, T, B, I, H, D, layers, states)
    "crnn": (0, 32, 32, 256, 256, 2, 2, False),
    "speech": (0, 200, 16, 80, 512, 1, 1, False),
    "kws": (0, 16, 1, 40, 128, 1, 1, True),
    "streamed": (0, 100, 64, 1024, 1024, 1, 1, False),
}
PLAN = ("cell", "t", "b", "i", "h", "d", "cs", "groups", "rows", "resident", "smem", "scratch", "launches", "ks")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else "unknown"
    except Exception:  # noqa: BLE001
        return "unknown"


def timed(fn, iters, rounds=5):
    import torch
    best = float("inf")
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        best = min(best, a.elapsed_time(b) * 1000.0 / iters)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    import torch
    from mnn_b200 import _capi
    from mnn_b200.backend import Runtime
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    rt = Runtime(0)   # adopts the current stream, so torch and the C ABI are ordered
    L, N = _capi.lib(), _capi.rnn_lib()
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    for name in args.cases.split(","):
        cell, T, B, I, H, D, layers, states = CASES[name]
        g = 4 if cell == 0 else 1
        rng = np.random.default_rng(1)
        dev = lambda *s: torch.from_numpy((rng.standard_normal(s) / np.sqrt(H)).astype(np.float32)).cuda()
        x = dev(T, B, I)
        lay = []
        for li in range(layers):
            i_in = I if li == 0 else D * H
            w, r, b = dev(D, g * H, i_in), dev(D, g * H, H), dev(D, g * H)
            h = C.c_void_p()
            assert N.mnnb200_rnn_create(rt._h, cell, C.byref(h)) == 0
            assert N.mnnb200_rnn_resize(h, T, B, i_in, H, D, int(states), int(states and cell == 0)) == 0, L.mnnb200_last_error()
            mm = C.c_void_p()
            assert L.mnnb200_matmul_create(rt._h, 1, T * B, i_in, D * g * H, 0, 1, 0, C.byref(mm)) == 0
            lay.append((h, mm, w, r, b, i_in))
        h0 = dev(D, B, H) if states else None
        c0 = dev(D, B, H) if states and cell == 0 else None
        ys = [torch.empty((T, D, B, H), device="cuda") for _ in range(layers)]
        yh, yc = torch.empty((D, B, H), device="cuda"), torch.empty((D, B, H), device="cuda")
        gates = torch.empty((T * B, D * g * H), device="cuda")

        def ours():
            inp = x
            for (h, _, w, r, b, _), y in zip(lay, ys):
                assert N.mnnb200_rnn_execute(h, p(inp), p(w), p(r), p(b), p(h0), p(c0), p(y), p(yh), p(yc)) == 0
                inp = y
        def proj():
            inp = x
            for (_, mm, w, _, b, _), y in zip(lay, ys):
                assert L.mnnb200_matmul_execute(mm, p(inp), p(w), p(b), p(gates)) == 0
                inp = y
        mod = (torch.nn.LSTM if cell == 0 else torch.nn.RNN)(I, H, num_layers=layers, bidirectional=D == 2).cuda()
        st = None
        if states:
            st = (h0.contiguous(), c0.contiguous()) if cell == 0 else h0.contiguous()
        with torch.no_grad():
            ref = lambda: mod(x, st)
            for f in (ours, proj, ref):
                f()
            torch.cuda.synchronize()
            t_ours, t_proj, t_ref = timed(ours, args.iters), timed(proj, args.iters), timed(ref, args.iters)
        f = (C.c_int * len(PLAN))()
        N.mnnb200_rnn_plan(lay[0][0], f, len(PLAN))
        print(json.dumps({"case": name, "cell": "LSTM" if cell == 0 else "RNN", "T": T, "B": B, "I": I, "H": H, "D": D,
                          "layers": layers, "us_per_execute": round(t_ours, 2), "us_per_step": round(t_ours / (T * layers), 3),
                          "us_projection": round(t_proj, 2), "us_recurrence": round(t_ours - t_proj, 2),
                          "us_cudnn": round(t_ref, 2), "cudnn_over_ours": round(t_ref / t_ours, 3),
                          "plan": dict(zip(PLAN, list(f))), "card": card()}), flush=True)
        for h, mm, *_ in lay:
            L.mnnb200_exec_destroy(h)
            L.mnnb200_exec_destroy(mm)


if __name__ == "__main__":
    main()
