"""Writes tests/golden/w4_linear_golden.npz: 4-bit LLM linear layers (MNN-LLM's --quant_bit 4 export) run through the real
reference CPU backend (`refdump_w4 linear`, oracle/refdump_w4.cpp).  Run from the repository root after oracle/build_ref.py and
`python -c "from oracle import w4_oracle; w4_oracle.build_refdump()"`.

Each case stores the packed weights exactly as ConvolutionCommon::load(..., forceInt8) hands them to a backend, the wire
{min, scale} pairs, the bias and the reference's fp32 output.  The cases cover one token (the single-quant decode form), 2-8
and >= 9 tokens, symmetric and asymmetric weights, per channel and blocks of 32 / 64 / 128, and oc on and off the fast int4
reorder condition of the AVX512 build (oc % 64 == 0), which selects the weightKernelSum rounding.

Recorded on an x86 host with AVX512-VNNI, so the reference ran _AVX512_MNNGemmInt8AddBiasScale_16x4_w4_Unit_VNNI.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from oracle import oracle as O  # noqa: E402

# tokens, ic, oc, bs (0: per channel), asym, bias, x range
CASES = [(1, 512, 128, 64, False, True, -1, 1), (1, 256, 96, 32, True, False, -1, 1), (1, 2048, 64, 128, True, True, 0.1, 2.0),
         (1, 300, 40, 0, False, True, -2, -0.5), (4, 256, 64, 32, False, False, -1, 1), (2, 512, 100, 64, True, True, -1, 1),
         (8, 384, 128, 128, True, False, -1, 1), (5, 128, 33, 0, True, True, -1, 1), (9, 512, 64, 64, False, True, -1, 1),
         (33, 256, 72, 128, True, True, -1, 1), (24, 1024, 128, 0, False, False, -1, 1), (17, 640, 96, 32, True, False, -1, 1),
         (1, 1024, 192, 0, True, True, -1, 1), (40, 512, 256, 64, True, True, -1, 1)]


def main():
    assert W.have_reference(), "build the reference and oracle/_ref/refdump_w4 first"
    rng = np.random.default_rng(404)
    out = {}
    for j, (tokens, ic, oc, bs, asym, hb, lo, hi) in enumerate(CASES):
        blocks = ic // bs if bs else 1
        x = rng.uniform(lo, hi, (tokens, ic)).astype(np.float32)
        q = rng.integers(-8, 8, (oc, ic)).astype(np.int8)
        alpha = rng.uniform(0.001, 0.01, (oc, blocks)).astype(np.float32)
        wmin = rng.uniform(-0.05, 0.05, (oc, blocks)).astype(np.float32) if asym else np.zeros(0, np.float32)
        bias = rng.uniform(-1, 1, oc).astype(np.float32) if hb else np.zeros(0, np.float32)
        wire = np.stack([wmin, alpha], 2).ravel() if asym else alpha.ravel()
        y = W.ref_linear(x, q, wire, asym=asym, bias=bias if hb else None, blocks=blocks)
        out.update({f"c{j}_x": x, f"c{j}_w": W.pack_w4(q), f"c{j}_alpha": alpha, f"c{j}_wmin": wmin, f"c{j}_bias": bias,
                    f"c{j}_y": y})
    out["n"] = len(CASES)
    np.savez_compressed(os.path.join(HERE, "w4_linear_golden.npz"), **out)
    print("w4_linear_golden.npz:", len(CASES), "cases")


if __name__ == "__main__":
    main()
