"""4-bit against 8-bit weights on one Qwen-1.8B layer's linears plus lm_head, K-blocked weight scales, in one process.

Shapes: 2048->6144 (+bias), 2048->2048, 2048->5504 x2, 5504->2048 and lm_head 2048->151936, asymmetric weights.  Prefill runs
4096 tokens through the five layer linears (lm_head on 8 tokens, the last token of each of 8 sequences); decode runs 1 token
through all six.  For each quant_block (64, 128) the 8-bit (mnnb200_linear_w8_create_blocked) and the 4-bit
(mnnb200_linear_w4_create_blocked) executions of the same shapes alternate, each window timed with CUDA events around the whole
set of layers; the median window is reported.  Prints one JSON line per (quant_block, regime) with the card name and power
limit: ms of each form, their ratio, and for decode the GB/s of each form with the weight bytes as stored (packed nibbles for
4 bits) plus the per-block alpha / wzero, the bias and the activations counted.

    python tools/w4_linear_bench.py [--reps 15]
"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.block_linear_bench import LAYER, H, V, card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("w4_linear_bench: no CUDA device (timings are only taken on the GPU)")
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
            sets = {"w8": [], "w4": []}
            wbytes = {"w8": 0.0, "w4": 0.0}
            macs = 0.0
            xs = {}
            for ic, oc, hb, t in shapes:
                q = rng.integers(-8, 8, (oc, ic), dtype=np.int8)
                blocks = ic // qb
                alpha_b = rng.uniform(0.001, 0.01, (oc, blocks)).astype(np.float32)
                wz_b = (alpha_b * rng.uniform(-8, 8, (oc, blocks))).astype(np.float32)
                bias = rng.uniform(-1, 1, oc).astype(np.float32) if hb else None
                key = (t, ic)
                if key not in xs:
                    xs[key] = torch.empty((t, ic), dtype=torch.float32, device="cuda").uniform_(-1, 1)
                macs += float(t) * ic * oc
                for form, w, bits in (("w8", q, 8), ("w4", None, 4)):
                    if bits == 4:
                        u = (q.reshape(-1).astype(np.int16) + 8).astype(np.uint8)
                        w = (u[0::2] << 4) | u[1::2]
                    op = Op(type="LinearW8", conv=dict(ic=ic, oc=oc), weight=w, wscale=alpha_b, wzero=wz_b, bias=bias, bits=bits)
                    x = Tensor((t, ic), "float", None, xs[key])
                    y = Tensor((t, oc), "float", None, torch.empty((t, oc), dtype=torch.float32, device="cuda"))
                    ex = be.onCreate([x], [y], op)
                    assert ex.onResize([x], [y]) == 0
                    sets[form].append((ex, x, y))
                    wbytes[form] += float(ic) * oc * bits / 8 + 8.0 * alpha_b.size + 4.0 * t * (ic + oc) + (4.0 * oc if hb else 0.0)
                del q

            def run(form):
                for ex, x, y in sets[form]:
                    assert ex.onExecute([x], [y]) == 0

            for _ in range(args.warmup):
                run("w8")
                run("w4")
            torch.cuda.synchronize()
            ms = {"w8": [], "w4": []}
            for _ in range(args.reps):
                for form in ("w8", "w4"):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(1 if T > 1 else 20):
                        run(form)
                    e1.record()
                    e1.synchronize()
                    ms[form].append(e0.elapsed_time(e1) / (1 if T > 1 else 20))
            med = {f: float(np.median(v)) for f, v in ms.items()}
            out = dict(card=name, power_limit=power, quant_block=qb, regime=regime, tokens=T,
                       w8_ms=round(med["w8"], 4), w4_ms=round(med["w4"], 4), w4_over_w8=round(med["w4"] / med["w8"], 3),
                       spread_w8_ms=[round(min(ms["w8"]), 4), round(max(ms["w8"]), 4)],
                       spread_w4_ms=[round(min(ms["w4"]), 4), round(max(ms["w4"]), 4)])
            if T == 1:
                out["w8_GBps"] = round(wbytes["w8"] / med["w8"] / 1e6, 1)
                out["w4_GBps"] = round(wbytes["w4"] / med["w4"] / 1e6, 1)
            else:
                out["w8_TMACs"] = round(macs / med["w8"] / 1e9, 1)
                out["w4_TMACs"] = round(macs / med["w4"] / 1e9, 1)
            print(json.dumps(out), flush=True)
            del sets
            torch.cuda.synchronize()
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
