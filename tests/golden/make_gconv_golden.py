"""Writes tests/golden/gconv_f32_golden.npz: grouped fp32 Convolution outputs recorded from the reference CPU backend
(oracle/_ref/refdump_gconv conv, built by build() where the reference sources are).

Each case's inputs are rebuilt from its seed by `case_inputs` (numpy's PCG64 generator, the same on every machine), so the
file holds only the outputs: all of them for small cases, a seeded subset of GCONV_KEEP positions for the larger ones.
Run: python tests/golden/make_gconv_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
PATH = os.path.join(ROOT, "tests", "golden", "gconv_f32_golden.npz")
GCONV_KEEP = 4096

# name: n, ic, oc, (ih, iw), kernel, stride, pads [t, l, b, r], dilation, group, inputCount, relu, relu6.  inputCount is what the
# op carries: ic (Express's _Conv) or ic / group (the TensorFlow form, where ConvolutionFloatFactory takes group = ic / inputCount)
CASES = {
    "resnext_stage1": (2, 128, 128, (14, 14), 3, 1, (1, 1, 1, 1), 1, 32, 128, 1, 0),
    "resnext_stage2_s2": (2, 256, 256, (15, 15), 3, 2, (1, 1, 1, 1), 1, 32, 256, 1, 0),
    "resnext_stage4": (2, 1024, 1024, (7, 7), 3, 1, (1, 1, 1, 1), 1, 32, 1024, 1, 0),
    "regnet_gw16": (2, 96, 96, (12, 12), 3, 1, (1, 1, 1, 1), 1, 6, 96, 1, 0),
    "regnet_gw16_s2": (2, 48, 48, (13, 11), 3, 2, (1, 1, 1, 1), 1, 3, 48, 0, 0),
    "shufflenet_g3_1x1": (2, 240, 240, (14, 14), 1, 1, (0, 0, 0, 0), 1, 3, 240, 1, 0),
    "shufflenet_g3_1x1_ic24": (2, 24, 60, (28, 28), 1, 1, (0, 0, 0, 0), 1, 3, 24, 1, 0),
    "alexnet_g2_k5": (2, 96, 256, (13, 13), 5, 1, (2, 2, 2, 2), 1, 2, 96, 1, 0),
    "depth_multiplier2": (2, 16, 32, (14, 14), 3, 1, (1, 1, 1, 1), 1, 16, 16, 0, 1),
    "dilation2_g8": (2, 64, 64, (12, 11), 3, 1, (2, 2, 2, 2), 2, 8, 64, 0, 0),
    "inputcount_per_group": (2, 48, 96, (10, 10), 3, 1, (1, 1, 1, 1), 1, 4, 12, 1, 0),
    "k3x5_s2x1_asym_pads_relu6": (2, 40, 80, (9, 13), (3, 5), (2, 1), (0, 2, 1, 1), 1, 5, 40, 0, 1),
    "ocg160_g2": (1, 40, 320, (6, 6), 3, 1, (1, 1, 1, 1), 1, 2, 40, 0, 0),
}


def pair(v):
    return tuple(v) if isinstance(v, (tuple, list)) else (v, v)


def case_inputs(name):
    """(x, w, b) of a case: x [n][ic][ih][iw], w [oc][ic / group][kh][kw], b [oc]"""
    n, ic, oc, (ih, iw), k, s, pads, d, group, _, _, relu6 = CASES[name]
    kh, kw = pair(k)
    rng = np.random.default_rng(sum(map(ord, name)))
    x = rng.standard_normal((n, ic, ih, iw)).astype(np.float32)
    fan = ic // group * kh * kw
    w = (rng.uniform(-1, 1, (oc, ic // group, kh, kw)) * (3 if relu6 else 1.2) / np.sqrt(fan)).astype(np.float32)
    b = rng.uniform(-0.5, 0.5, oc).astype(np.float32)
    return x, w, b


def load():
    """{name: (y or None, flat indices or None, y shape)}"""
    z = np.load(PATH)
    return {name: (z[name + "_y"], z[name + "_idx"] if name + "_idx" in z.files else None, tuple(z[name + "_shape"]))
            for name in CASES}


def main():
    sys.path.insert(0, ROOT)
    from oracle import gconv_oracle as G
    out = {}
    for name, (n, ic, oc, hw, k, s, pads, d, group, input_count, relu, relu6) in CASES.items():
        x, w, b = case_inputs(name)
        y = G.ref_gconv(x, w, b, group, input_count, s, pads, d, bool(relu), bool(relu6))
        out[name + "_shape"] = np.array(y.shape, np.int32)
        if y.size > GCONV_KEEP:
            idx = np.sort(np.random.default_rng(len(name)).choice(y.size, GCONV_KEEP, replace=False)).astype(np.int32)
            out[name + "_idx"] = idx
            out[name + "_y"] = y.reshape(-1)[idx]
        else:
            out[name + "_y"] = y.reshape(-1)
        print(name, y.shape)
    np.savez_compressed(PATH, **out)
    print("wrote", PATH, os.path.getsize(PATH), "bytes")


if __name__ == "__main__":
    main()
