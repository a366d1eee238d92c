"""LayerNorm / RMSNorm and fused RoPE at Qwen-1.8B shapes through the C ABI: device time per call and achieved GB/s.

Cases, each at decode (1 token) and prefill (4096 tokens): the RMSNorm over hidden 2048 (gamma and beta), the residual RMSNorm
(sum = x + r, y = norm(sum)), RoPE 16 x 128 without GQA and GQA 12 / 2 x 128, both rotating the whole head, and RoPE 16 / 8 x 128
with Qwen3's q / k RMSNorm.  Every call is timed as a window of back-to-back launches between CUDA events (median of --reps
windows of --calls calls).  GB/s counts the algorithmic bytes: norm 8 B per element (+ 8 B per gamma / beta element), residual
16 B per element, RoPE 8 B per q / k element + 8 B per cos / sin element.  The HBM bound is printed at the H100 SXM data sheet's
3.35 TB/s; `launch_floor_us` is the same window of a one-element torch add, for the decode calls.  One JSON line per case, with the
card name and power limit.

    python tools/llm_ops_bench.py [--reps 9] [--calls 200]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.block_linear_bench import card  # noqa: E402

HBM = 3.35e12


def timed(fn, reps, calls):
    import torch
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(calls):
            fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) * 1e3 / calls)
    times.sort()
    return times[len(times) // 2], times[0], times[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--calls", type=int, default=200)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("llm_ops_bench: no CUDA device (timings are only taken on the GPU)")
    from mnn_b200 import _capi
    from mnn_b200.backend import Runtime
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    be = Runtime(0).onCreate()
    rt, L, core = be.runtime._h, _capi.llm_lib(), _capi.lib()
    name, power = card()
    rng = np.random.default_rng(0)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()
    p = lambda t: C.c_void_p(t.data_ptr())
    one = torch.zeros(1, device="cuda")
    floor = timed(lambda: one.add_(0), args.reps, args.calls)[0]
    H = 2048
    gamma, beta = rng.uniform(0.5, 1.5, H).astype(np.float32), np.zeros(H, np.float32)
    for regime, T in (("decode", 1), ("prefill", 4096)):
        x, r = dev(rng.standard_normal((T, H))), dev(rng.standard_normal((T, H)))
        s, y = torch.empty_like(x), torch.empty_like(x)
        h = C.c_void_p()
        _capi.check(L.mnnb200_layernorm_f32_create(rt, H, 1e-6, 1, gamma.ctypes.data, beta.ctypes.data, H, C.byref(h)), "create")
        _capi.check(L.mnnb200_layernorm_f32_resize(h, T), "resize")
        cases = [("rmsnorm", lambda: L.mnnb200_layernorm_f32_execute(h, p(x), None, None, p(y)), 8.0 * T * H + 8.0 * H),
                 ("residual_rmsnorm", lambda: L.mnnb200_layernorm_f32_execute(h, p(x), p(r), p(s), p(y)), 16.0 * T * H + 8.0 * H)]
        handles = [h]
        for tag, heads, kvh, norm in (("rope_16x128", 16, 16, False), ("rope_gqa_12_2x128", 12, 2, False),
                                      ("rope_qk_rmsnorm_16_8x128", 16, 8, True)):
            hd = 128
            q, k = dev(rng.standard_normal((T, heads * hd))), dev(rng.standard_normal((T, kvh * hd)))
            cs, sn = dev(rng.uniform(-1, 1, (T, hd))), dev(rng.uniform(-1, 1, (T, hd)))
            qo, ko = torch.empty_like(q), torch.empty_like(k)
            g = np.ones(hd, np.float32)
            tab = _capi.RopeNorm(g.ctypes.data, None, hd, 1e-6, 1)
            hr = C.c_void_p()
            _capi.check(L.mnnb200_rope_f32_create(rt, heads, kvh, hd, 0, C.byref(tab) if norm else None,
                                                  C.byref(tab) if norm else None, C.byref(hr)), "rope create")
            _capi.check(L.mnnb200_rope_f32_resize(hr, T, heads * hd, kvh * hd), "rope resize")
            handles.append(hr)
            bytes_ = 8.0 * T * (heads + kvh) * hd + 8.0 * T * hd
            keep = (q, k, cs, sn, qo, ko)
            cases.append((tag, (lambda hr=hr, keep=keep: L.mnnb200_rope_f32_execute(hr, *(p(t) for t in keep))), bytes_))
        for tag, fn, nbytes in cases:
            assert fn() == 0, core.mnnb200_last_error()
            med, lo, hi = timed(fn, args.reps, args.calls)
            print(json.dumps({"case": tag, "regime": regime, "tokens": T, "us_per_call": round(med, 3), "us_min": round(lo, 3),
                              "us_max": round(hi, 3), "bytes": nbytes, "GBps": round(nbytes / med * 1e-3, 1),
                              "hbm_bound_us": round(nbytes / HBM * 1e6, 3), "launch_floor_us": round(floor, 3),
                              "card": name, "power_limit": power}), flush=True)
        for hh in handles:
            core.mnnb200_exec_destroy(hh)


if __name__ == "__main__":
    main()
