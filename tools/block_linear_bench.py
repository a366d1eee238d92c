"""Blocked (quant_block) against per-channel int8 weight scales on one Qwen-1.8B layer's linears plus lm_head, in one process.

Shapes: 2048->6144 (+bias), 2048->2048, 2048->5504 x2, 5504->2048 and lm_head 2048->151936, asymmetric weights.  Prefill runs
4096 tokens through the five layer linears (lm_head on 8 tokens, the last token of each of 8 sequences); decode runs 1 token
through all six.  For each quant_block (64, 128) the per-channel and the blocked executions of the same weights alternate, each
window timed with CUDA events around the whole set of layers; the median window is reported.  Prints one JSON line per
(quant_block, regime) with the card name and power limit: ms of each form, their ratio, and for decode the GB/s of each form
with the per-block alpha / wzero bytes counted.

    python tools/block_linear_bench.py [--reps 15]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

H, F, V = 2048, 5504, 151936
LAYER = [(H, 3 * H, True), (H, H, False), (H, F, False), (H, F, False), (F, H, False)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in q.split(","))
        return name, power
    except Exception as e:          # the timing itself needs no nvidia-smi
        return f"unknown ({e})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("block_linear_bench: no CUDA device (timings are only taken on the GPU)")
    from mnn_b200.backend import Op, Runtime, Tensor
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    rt = Runtime(0)
    be = rt.onCreate()
    name, power = card()
    rng = np.random.default_rng(0)
    for qb in (64, 128):
        for regime, T in (("prefill", 4096), ("decode", 1)):
            shapes = [(ic, oc, hb, T) for ic, oc, hb in LAYER] + [(H, V, False, 8 if T > 1 else 1)]
            sets = {"per_channel": [], "blocked": []}
            wbytes = {"per_channel": 0.0, "blocked": 0.0}
            macs = 0.0
            xs = {}
            for ic, oc, hb, t in shapes:
                wq = rng.integers(-128, 128, (oc, ic), dtype=np.int8)
                blocks = ic // qb
                alpha_b = rng.uniform(0.001, 0.01, (oc, blocks)).astype(np.float32)
                wz_b = (alpha_b * rng.uniform(-8, 8, (oc, blocks))).astype(np.float32)
                bias = rng.uniform(-1, 1, oc).astype(np.float32) if hb else None
                key = (t, ic)
                if key not in xs:
                    xs[key] = torch.empty((t, ic), dtype=torch.float32, device="cuda").uniform_(-1, 1)
                macs += float(t) * ic * oc
                for form, al, wz in (("per_channel", alpha_b[:, 0].copy(), wz_b[:, 0].copy()), ("blocked", alpha_b, wz_b)):
                    op = Op(type="LinearW8", conv=dict(ic=ic, oc=oc), weight=wq, wscale=al, wzero=wz, bias=bias)
                    x = Tensor((t, ic), "float", None, xs[key])
                    y = Tensor((t, oc), "float", None, torch.empty((t, oc), dtype=torch.float32, device="cuda"))
                    ex = be.onCreate([x], [y], op)
                    assert ex.onResize([x], [y]) == 0
                    sets[form].append((ex, x, y))
                    wbytes[form] += float(ic) * oc + 8.0 * al.size + 4.0 * t * (ic + oc) + (4.0 * oc if hb else 0.0)

            def run(form):
                for ex, x, y in sets[form]:
                    assert ex.onExecute([x], [y]) == 0

            for _ in range(args.warmup):
                run("per_channel")
                run("blocked")
            torch.cuda.synchronize()
            ms = {"per_channel": [], "blocked": []}
            for _ in range(args.reps):
                for form in ("per_channel", "blocked"):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(1 if T > 1 else 20):
                        run(form)
                    e1.record()
                    e1.synchronize()
                    ms[form].append(e0.elapsed_time(e1) / (1 if T > 1 else 20))
            med = {f: float(np.median(v)) for f, v in ms.items()}
            out = dict(card=name, power_limit=power, quant_block=qb, regime=regime, tokens=T,
                       per_channel_ms=round(med["per_channel"], 4), blocked_ms=round(med["blocked"], 4),
                       blocked_over_per_channel=round(med["blocked"] / med["per_channel"], 3))
            if T == 1:
                out["per_channel_GBps"] = round(wbytes["per_channel"] / med["per_channel"] / 1e6, 1)
                out["blocked_GBps"] = round(wbytes["blocked"] / med["blocked"] / 1e6, 1)
            else:
                out["per_channel_TMACs"] = round(macs / med["per_channel"] / 1e9, 1)
                out["blocked_TMACs"] = round(macs / med["blocked"] / 1e9, 1)
            print(json.dumps(out), flush=True)
            del sets
            torch.cuda.synchronize()
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
