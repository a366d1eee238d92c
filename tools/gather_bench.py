#!/usr/bin/env python3
"""The gathers and the broadcast float MatMul at sizes users run, one JSON line per case, each with:
  us            device time per launch (CUDA events around --iters back-to-back launches after --warmup, best of --rounds);
  bytes / flops gathers: the gathered rows read once, the output written once and the indices read once (4-byte elements);
                MatMul: 2 e l h per output batch, from shapes;
  bound_share   gathers: bytes / 3.35 TB/s (H100 SXM HBM3, data sheet at 700 W; the bound, not a reached figure) over the time;
                MatMul: flops / 495 TFLOP/s (dense TF32, same data sheet) over the time;
  torch_us      in the same process, alternating with the kernel: torch.index_select (Gather), torch.gather (GatherElements) or
                torch.matmul (default TF32 off: a yardstick for speed only) on the same tensors;
  card          name and power limit, read in the same call.
Usage: python tools/gather_bench.py [--iters 200] [--warmup 20] [--rounds 5]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BPS = 3.35e12
TF32_FLOPS = 495e12


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
    assert torch.cuda.is_available(), "gather_bench needs an H100 (there is no CPU path)"
    from mnn_b200 import _capi
    from mnn_b200.backend import Runtime
    rt = Runtime(0).onCreate().runtime
    G, L = _capi.gather_lib(), _capi.lib()
    who = card()
    print(json.dumps({"card": who}))
    p = lambda t: C.c_void_p(t.data_ptr())   # noqa: E731
    arr = lambda v: (C.c_int * max(len(v), 1))(*v)   # noqa: E731

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

    def report(name, ours, theirs, extra, nbytes=None, flops=None):
        t_ours, t_torch = [], []
        for _ in range(a.rounds):
            t_ours.append(timed(ours))
            t_torch.append(timed(theirs))
        us = min(t_ours)
        share = nbytes / HBM_BPS if nbytes else flops / TF32_FLOPS
        out = dict(case=name, us=round(us, 2), us_spread=[round(min(t_ours), 2), round(max(t_ours), 2)],
                   bound="hbm" if nbytes else "tf32", bound_share=round(share / (us * 1e-6), 3), torch_us=round(min(t_torch), 2),
                   card=who, **extra)
        if nbytes:
            out["bytes"] = nbytes
        else:
            out["flops"] = flops
        print(json.dumps(out))

    def gather_case(name, mode, params, idx, axis, torch_fn, out_shape):
        h = C.c_void_p()
        _capi.check(G.mnnb200_gather_create(rt._h, mode, C.byref(h)), "gather_create")
        _capi.check(G.mnnb200_gather_resize(h, arr(params.shape), params.dim(), arr(idx.shape), idx.dim(), axis), "gather_resize")
        y = torch.empty(out_shape, dtype=params.dtype, device="cuda")
        pp, ip, yp = p(params), p(idx), p(y)
        ours = lambda: G.mnnb200_gather_execute(h, pp, ip, yp)   # noqa: E731
        ours()
        torch.cuda.synchronize()
        ref = torch_fn()
        assert torch.equal(y, ref.reshape(out_shape)), name
        f = (C.c_int * 8)()
        _capi.check(G.mnnb200_gather_plan(h, f, 8), "gather_plan")
        nbytes = 2 * y.numel() * 4 + idx.numel() * 4
        report(name, ours, torch_fn, dict(path=f[1], grid=f[2], slices_per_tile=f[4]), nbytes=nbytes)
        L.mnnb200_exec_destroy(h)

    emb = torch.randn(30522, 768, device="cuda")
    for b, s in ((32, 128), (8, 512)):
        ids = torch.randint(0, 30522, (b, s), dtype=torch.int32, device="cuda")
        ids64 = ids.long().reshape(-1)
        gather_case(f"bert_base_embedding_{b}x{s}", 0, emb, ids, 0, lambda: torch.index_select(emb, 0, ids64), (b, s, 768))
    x = torch.randn(32, 197, 768, device="cuda")
    zero = torch.zeros(1, dtype=torch.int32, device="cuda")
    zero64 = zero.long()
    gather_case("vit_class_token_32x197x768", 0, x, zero, 1, lambda: torch.index_select(x, 1, zero64), (32, 1, 768))
    scores = torch.randn(32, 1000, 4096, device="cuda")
    top = torch.randint(0, 4096, (32, 1000, 100), dtype=torch.int32, device="cuda")
    top64 = top.long()
    gather_case("topk_gather_elements_32x1000x4096_k100", 2, scores, top, 2, lambda: torch.gather(scores, 2, top64),
                (32, 1000, 100))

    # BERT-base attention at batch 32, 12 heads, S 128, head 64: QK^T (adjY) and PV
    q = torch.randn(32, 12, 128, 64, device="cuda")
    k = torch.randn(32, 12, 128, 64, device="cuda")
    pr = torch.softmax(torch.randn(32, 12, 128, 128, device="cuda"), -1)
    for name, A, B, tb, e, l, hh, fn in (("bert_base_qk_t_b32_h12_s128", q, k, 1, 128, 64, 128, lambda: torch.matmul(q, k.transpose(-1, -2))),
                                         ("bert_base_pv_b32_h12_s128", pr, q, 0, 128, 128, 64, lambda: torch.matmul(pr, q))):
        h = C.c_void_p()
        nd = (32, 12)
        _capi.check(L.mnnb200_matmul_create_broadcast(rt._h, 2, arr(nd), arr(nd), arr(nd), e, l, hh, 0, tb, C.byref(h)), "matmul")
        c = torch.empty(32, 12, e, hh, device="cuda")
        ap_, bp, cp = p(A), p(B), p(c)
        ours = lambda: L.mnnb200_matmul_execute(h, ap_, bp, None, cp)   # noqa: E731
        ours()
        torch.cuda.synchronize()
        ref = fn()
        err = float((c - ref).abs().max() / ref.abs().max())
        report(name, ours, fn, dict(rel_err_vs_torch=err), flops=2.0 * 32 * 12 * e * l * hh)
        L.mnnb200_exec_destroy(h)


if __name__ == "__main__":
    main()
