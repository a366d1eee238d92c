"""Writes tests/golden/deconv_f32_golden.npz: fp32 Deconvolution outputs recorded from the reference CPU backend
(oracle/_ref/refdump_deconv deconv, built by build() where the reference sources are).

Each case's inputs are rebuilt from its seed by `case_inputs` (numpy's PCG64 generator, the same on every machine), so the
file holds only the outputs: all of them for small cases, a seeded subset of DECONV_KEEP positions for the larger ones.
Run: python tests/golden/make_deconv_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
PATH = os.path.join(ROOT, "tests", "golden", "deconv_f32_golden.npz")
DECONV_KEEP = 4096

# name: n, ic, oc, (ih, iw), k, stride, pads [t, l, b, r], dilation, out_pads, same, output shape (None: from the op), depthwise,
# relu, relu6
CASES = {
    "k2_s2": (2, 8, 6, (5, 7), 2, 2, (0, 0, 0, 0), 1, (0, 0), 0, None, 0, 0, 0),
    "k3_s2_p1_outpad1": (2, 7, 9, (6, 5), 3, 2, (1, 1, 1, 1), 1, (1, 1), 0, None, 0, 0, 0),
    "k4_s2_p1": (2, 16, 12, (8, 6), 4, 2, (1, 1, 1, 1), 1, (0, 0), 0, None, 0, 0, 0),
    "k16_s8_p4": (1, 5, 21, (4, 5), 16, 8, (4, 4, 4, 4), 1, (0, 0), 0, None, 0, 0, 0),
    "k3_s2_d2": (2, 6, 10, (7, 6), 3, 2, (1, 1, 1, 1), 2, (0, 0), 0, None, 0, 0, 0),
    "k1_s2": (2, 9, 7, (6, 5), 1, 2, (0, 0, 0, 0), 1, (0, 0), 0, None, 0, 0, 0),
    "k3_s2_same": (2, 8, 6, (5, 7), 3, 2, (0, 0, 0, 0), 1, (0, 0), 1, None, 0, 0, 0),
    "k3_s2_output_shape": (2, 8, 6, (5, 7), 3, 2, (0, 0, 0, 0), 1, (0, 0), 1, (10, 13), 0, 0, 0),
    "k4_s2_asym_pads": (2, 6, 5, (6, 6), 4, 2, (0, 1, 2, 1), 1, (0, 0), 0, None, 0, 0, 0),
    "k4_s2_p1_relu": (2, 12, 10, (6, 7), 4, 2, (1, 1, 1, 1), 1, (0, 0), 0, None, 0, 1, 0),
    "k3_s2_p1_relu6": (2, 12, 10, (6, 7), 3, 2, (1, 1, 1, 1), 1, (1, 1), 0, None, 0, 0, 1),
    "dw_k4_s2_p1": (2, 16, 16, (7, 6), 4, 2, (1, 1, 1, 1), 1, (0, 0), 0, None, 1, 1, 0),
}


def case_inputs(name):
    """(x, w, b) of a case: x [n][ic][ih][iw], w [ic][oc][kh][kw] ([c][kh][kw] depthwise), b [oc]"""
    n, ic, oc, (ih, iw), k, *_, dw, _, relu6 = CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    x = rng.standard_normal((n, ic, ih, iw)).astype(np.float32)
    w = (rng.uniform(-1, 1, (ic, k, k) if dw else (ic, oc, k, k)) * (3 if relu6 else 1.2) / np.sqrt(ic * k * k)).astype(np.float32)
    b = rng.uniform(-0.5, 0.5, oc).astype(np.float32)
    return x, w, b


def begin_pads(name, out_hw):
    """ConvolutionCommon::convolutionTransposePad: (top, left) for the output size MNN's shape inference gave"""
    n, ic, oc, (ih, iw), k, s, pads, *_ = CASES[name]
    if CASES[name][9]:
        return ((ih - 1) * s + k - out_hw[0]) // 2, ((iw - 1) * s + k - out_hw[1]) // 2
    return pads[0], pads[1]


def load():
    """{name: (y or None, flat indices or None, y shape)}"""
    z = np.load(PATH)
    return {name: (z[name + "_y"], z[name + "_idx"] if name + "_idx" in z.files else None, tuple(z[name + "_shape"]))
            for name in CASES}


def main():
    sys.path.insert(0, ROOT)
    from oracle import deconv_oracle as D
    out = {}
    for name, (n, ic, oc, hw, k, s, pads, d, op, same, shape, dw, relu, relu6) in CASES.items():
        x, w, b = case_inputs(name)
        y = D.ref_deconv(x, w, b, s, pads, d, op, bool(same), shape, bool(dw), bool(relu), bool(relu6))
        out[name + "_shape"] = np.array(y.shape, np.int32)
        if y.size > DECONV_KEEP:
            idx = np.sort(np.random.default_rng(len(name)).choice(y.size, DECONV_KEEP, replace=False)).astype(np.int32)
            out[name + "_idx"] = idx
            out[name + "_y"] = y.reshape(-1)[idx]
        else:
            out[name + "_y"] = y.reshape(-1)
        print(name, y.shape)
    np.savez_compressed(PATH, **out)
    print("wrote", PATH, os.path.getsize(PATH), "bytes")


if __name__ == "__main__":
    main()
