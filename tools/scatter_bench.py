#!/usr/bin/env python3
"""ScatterNd and ScatterElements at sizes users run, one JSON line per case, each with:
  us            device time per launch (CUDA events around --iters back-to-back executes after --warmup, best of --rounds);
  bytes         from shapes: y written once, data read once (when the op has data), updates and indices read once;
  bound_share   bytes / 3.35 TB/s (H100 SXM HBM3, data sheet at 700 W; the bound, not a reached figure) over the time;
  torch_us      in the same process, alternating with the kernel: index_put_ (ScatterNd) or scatter_add_ (ScatterElements ADD)
                on the same tensors, after the same copy or zero fill of the output;
  torch_det_us  the same under torch.use_deterministic_algorithms(True);
  plan          the execution's path, sort passes, launches and grid;
  card          name and power limit, read in the same call.
Cases: a PointPillars BEV canvas (about 12,000 pillars x 64 channels into 496 x 432, batch 1 and 4, padding pillars at cell 0),
a KV-cache row write (1 and 512 rows into [4096, 4096]), a GNN scatter-add (1 M edges x 64 features into 100 k nodes, uniform
and with one hub node taking 10 % of the edges) and a histogram (1 M scalar updates into 1,000 bins).
Usage: python tools/scatter_bench.py [--iters 50] [--warmup 5] [--rounds 5]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BPS = 3.35e12
PLAN = ("mode", "reduction", "n", "s", "r", "x", "path", "passes", "launches", "vec", "init_vec", "grid")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError, IndexError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "scatter_bench needs an H100 (there is no CPU path)"
    torch.cuda.set_stream(torch.cuda.Stream())        # one stream, current for torch and adopted by the runtime
    from mnn_b200 import _capi
    from mnn_b200.backend import Runtime
    rt = Runtime(0).onCreate().runtime
    S, L = _capi.scatter_lib(), _capi.lib()
    who = card()
    print(json.dumps({"card": who}))
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None   # noqa: E731
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

    def case(name, mode, red, out_shape, idx, upd, data, axis, torch_fn):
        h = C.c_void_p()
        _capi.check(S.mnnb200_scatter_create(rt._h, mode, red, int(data is not None), C.byref(h)), "scatter_create")
        _capi.check(S.mnnb200_scatter_resize(h, arr(out_shape), len(out_shape), arr(idx.shape), idx.dim(), arr(upd.shape), upd.dim(),
                                             axis, 0), "scatter_resize")
        y = torch.empty(out_shape, dtype=torch.float32, device="cuda")
        dp, ip, up, yp = p(data), p(idx), p(upd), p(y)
        ours = lambda: S.mnnb200_scatter_execute(h, dp, ip, up, yp)   # noqa: E731
        ours()
        torch.cuda.synchronize()
        ref = torch_fn()
        diff = float((y - ref).abs().max() / ref.abs().max().clamp_min(1e-30))
        f = (C.c_int * len(PLAN))()
        _capi.check(S.mnnb200_scatter_plan(h, f, len(PLAN)), "scatter_plan")
        pl = dict(zip(PLAN, f))
        t_ours, t_torch, t_det = [], [], []
        for _ in range(a.rounds):
            t_ours.append(timed(ours))
            t_torch.append(timed(torch_fn))
            torch.use_deterministic_algorithms(True)
            try:
                t_det.append(timed(torch_fn))
            finally:
                torch.use_deterministic_algorithms(False)
        us = min(t_ours)
        nbytes = 4 * (y.numel() * (2 if data is not None else 1) + upd.numel() + idx.numel())
        print(json.dumps(dict(case=name, us=round(us, 2), us_spread=[round(min(t_ours), 2), round(max(t_ours), 2)], bytes=nbytes,
                              bound="hbm", bound_share=round(nbytes / HBM_BPS / (us * 1e-6), 3), torch_us=round(min(t_torch), 2),
                              torch_det_us=round(min(t_det), 2), max_rel_diff_vs_torch=diff,
                              plan={k: pl[k] for k in ("path", "passes", "launches", "vec", "grid", "x")}, card=who)))
        L.mnnb200_exec_destroy(h)

    g = torch.Generator(device="cuda")
    g.manual_seed(0)
    # PointPillars: pillar vectors into a zero BEV canvas [B * H * W, C]; pillars past the real ones pad at cell 0
    H, W, Ch = 496, 432, 64
    for b in (1, 4):
        pillars, real = 12000 * b, 9000 * b
        cell = torch.zeros(pillars, 1, dtype=torch.int32, device="cuda")
        cell[:real, 0] = torch.randperm(b * H * W, device="cuda", generator=g)[:real].int()
        feats = torch.relu(torch.randn(pillars, Ch, device="cuda", generator=g))
        canvas = torch.empty(b * H * W, Ch, device="cuda")
        c64 = cell.long().reshape(-1)
        # the padding pillars go first in torch's write, so the last real writer of cell 0 wins as in the op
        def pillars_torch(canvas=canvas, c64=c64, feats=feats):
            canvas.zero_()
            return canvas.index_put_((c64,), feats)
        case(f"pointpillars_canvas_b{b}", 0, -1, (b * H * W, Ch), cell, feats, None, 0, pillars_torch)
    # KV cache: rows written into a copy of the cache
    cache = torch.randn(4096, 4096, device="cuda", generator=g)
    for rows in (1, 512):
        pos = torch.randperm(4096, device="cuda", generator=g)[:rows].int().reshape(rows, 1)
        new = torch.randn(rows, 4096, device="cuda", generator=g)
        out = torch.empty_like(cache)
        p64 = pos.long().reshape(-1)
        def kv_torch(out=out, p64=p64, new=new):
            out.copy_(cache)
            return out.index_put_((p64,), new)
        case(f"kv_cache_write_{rows}_rows", 0, -1, (4096, 4096), pos, new, cache, 0, kv_torch)
    # GNN mean aggregation's sum: messages of 1 M edges added into 100 k nodes (ScatterElements ADD on axis 0)
    V, E, F = 100_000, 1_000_000, 64
    for hub in (False, True):
        dst = torch.randint(0, V, (E,), device="cuda", generator=g)
        if hub:
            dst[torch.randperm(E, device="cuda", generator=g)[:E // 10]] = 0
        idx = dst.int().reshape(E, 1).expand(E, F).contiguous()
        msg = torch.randn(E, F, device="cuda", generator=g)
        base = torch.zeros(V, F, device="cuda")
        out = torch.empty(V, F, device="cuda")
        i64 = idx.long()
        def gnn_torch(out=out, i64=i64, msg=msg, base=base):
            out.copy_(base)
            return out.scatter_add_(0, i64, msg)
        case("gnn_scatter_add_1m_edges_64f" + ("_hub10pct" if hub else "_uniform"), 1, 0, (V, F), idx, msg, base, 0, gnn_torch)
    # a histogram: 1 M scalar updates into 1,000 bins
    bins = torch.randint(0, 1000, (1_000_000,), device="cuda", generator=g).int()
    w = torch.rand(1_000_000, device="cuda", generator=g)
    zero = torch.zeros(1000, device="cuda")
    hist = torch.empty(1000, device="cuda")
    b64 = bins.long()
    def hist_torch():
        hist.copy_(zero)
        return hist.scatter_add_(0, b64, w)
    case("histogram_1m_into_1000_bins", 1, 0, (1000,), bins, w, zero, 0, hist_torch)


if __name__ == "__main__":
    main()
