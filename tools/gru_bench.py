"""GRU through the C ABI (mnnb200_gru_*) over a grid of sizes: linear_before_reset 0 and 1, D 1 and 2, H in {64, 128, 256,
512, 1024}, B in {1, 8, 64}, T 100, I = H.  For linear_before_reset 1 (torch's form) torch.nn.GRU in fp32 on cuDNN (TF32 off)
runs the same layer in the same process.  One JSON line per row: device µs per execute (CUDA events over back-to-back executes,
best of 3 rounds), µs per step, the plan (cluster size, R resident or streamed, threads per dot product), cuDNN's µs, card name
and power limit.  --lbr / --d / --h / --b take comma lists to run a part of the grid."""
import argparse
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.rnn_bench import card, timed  # noqa: E402

PLAN = ("lbr", "t", "b", "i", "h", "d", "cs", "groups", "rows", "resident", "smem", "scratch", "launches", "ks")


def ints(s):
    return [int(v) for v in s.split(",")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lbr", default="0,1")
    ap.add_argument("--d", default="1,2")
    ap.add_argument("--h", default="64,128,256,512,1024")
    ap.add_argument("--b", default="1,8,64")
    ap.add_argument("--t", type=int, default=100)
    args = ap.parse_args()
    import numpy as np
    import torch
    from mnn_b200 import _capi
    from mnn_b200.backend import Runtime
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    rt = Runtime(0)   # adopts the current stream, so torch and the C ABI are ordered
    L, G = _capi.lib(), _capi.gru_lib()
    p = lambda t: C.c_void_p(t.data_ptr())
    name = card()
    T = args.t
    for lbr in ints(args.lbr):
        for D in ints(args.d):
            for H in ints(args.h):
                for B in ints(args.b):
                    I = H
                    rng = np.random.default_rng(1)
                    dev = lambda *s: torch.from_numpy((rng.standard_normal(s) / np.sqrt(H)).astype(np.float32)).cuda()
                    x = dev(T, B, I)
                    params = []
                    for _ in range(D):
                        params += [dev(I + H, 2 * H), dev(1, 2 * H), dev(I + H, H), dev(1, H), dev(1, 3 * H)]
                    arr = (C.c_void_p * len(params))(*[t.data_ptr() for t in params])
                    y, yh = torch.empty((T, D, B, H), device="cuda"), torch.empty((D, B, H), device="cuda")
                    h = C.c_void_p()
                    assert G.mnnb200_gru_create(rt._h, lbr, C.byref(h)) == 0
                    assert G.mnnb200_gru_resize(h, T, B, I, H, D, 0) == 0, L.mnnb200_last_error()
                    ours = lambda: G.mnnb200_gru_execute(h, p(x), arr, None, p(y), p(yh))
                    ours()
                    torch.cuda.synchronize()
                    t1 = timed(ours, 1, rounds=1)
                    iters = int(max(2, min(20, 200000.0 / max(t1, 1.0))))
                    t_ours = timed(ours, iters, rounds=3)
                    row = {"lbr": lbr, "T": T, "B": B, "I": I, "H": H, "D": D, "us_per_execute": round(t_ours, 2),
                           "us_per_step": round(t_ours / T, 3)}
                    if lbr == 1:
                        mod = torch.nn.GRU(I, H, bidirectional=D == 2).cuda()
                        with torch.no_grad():
                            ref = lambda: mod(x)
                            ref()
                            torch.cuda.synchronize()
                            t_ref = timed(ref, iters, rounds=3)
                        row.update(us_cudnn=round(t_ref, 2), cudnn_over_ours=round(t_ref / t_ours, 3))
                    f = (C.c_int * len(PLAN))()
                    G.mnnb200_gru_plan(h, f, len(PLAN))
                    pl = dict(zip(PLAN, list(f)))
                    row.update(plan={k: pl[k] for k in ("cs", "groups", "rows", "resident", "ks", "smem")},
                               r="resident" if pl["resident"] else "streamed", card=name)
                    print(json.dumps(row), flush=True)
                    L.mnnb200_exec_destroy(h)


if __name__ == "__main__":
    main()
