"""Writes tests/golden/interp_f32_golden.npz: fp32 Interp outputs recorded from the reference CPU backend (oracle/_ref/refdump_interp
op, built by build() where the reference sources are).

Each case's input is rebuilt from its seed by `case_inputs` (numpy's PCG64 generator, the same on every machine).  The outputs are
bit-exact targets, so the file holds only their shape and the sha256 of their fp32 bytes.
Run: python tests/golden/make_interp_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
PATH = os.path.join(ROOT, "tests", "golden", "interp_f32_golden.npz")

# the coordinate-transform forms: (ctm, alignCorners, halfPixelCenters)
FORMS = {"notset_align": ("NotSet", 1, 0), "notset_half": ("NotSet", 0, 1), "notset": ("NotSet", 0, 0),
         "align": ("AlignCorners", 0, 0), "half": ("HalfPixels", 0, 0), "pytorch": ("PytorchHalfPixels", 0, 0),
         "asym": ("Asymmetric", 0, 0), "tfhalf": ("TensorflowHalfPixels", 0, 0)}
# (n, c, (ih, iw), (oh, ow)): integer x2 with ow % 4 != 0 and batch 2, fractional up, 0.5x down, 1x1 -> HxW, HxW -> 1x1, x4,
# fractional down, fractional up; channel counts not a multiple of 4 (the CPU pads NC4HW4) in most
SHAPES = [(2, 5, (7, 9), (14, 18)), (1, 6, (9, 10), (17, 23)), (1, 8, (32, 24), (16, 12)), (2, 3, (1, 1), (16, 16)),
          (1, 5, (9, 7), (1, 1)), (1, 4, (16, 16), (64, 64)), (2, 7, (11, 13), (8, 10)), (1, 3, (10, 10), (25, 31))]
TYPES = {1: "nearest", 2: "bilinear", 3: "cubic", 4: "round"}


def _cases():
    cases = {}
    for ti, (t, tname) in enumerate(TYPES.items()):
        for fi, (fname, (ctm, align, half)) in enumerate(FORMS.items()):
            n, c, ihw, ohw = SHAPES[(fi + 3 * ti) % len(SHAPES)]
            cases[f"{tname}_{fname}"] = dict(n=n, c=c, in_hw=ihw, resize_type=t, ctm=ctm, align=align, half=half, out_hw=ohw)
    # the other ways to give the output size, and an NHWC input
    cases["bilinear_scales_input"] = dict(n=1, c=4, in_hw=(10, 10), resize_type=2, ctm="HalfPixels", align=0, half=0,
                                          out_hw=(0, 0), scales=(2.0, 1.5))
    cases["cubic_scales_input"] = dict(n=1, c=3, in_hw=(6, 8), resize_type=3, ctm="NotSet", align=0, half=0, out_hw=(0, 0),
                                       scales=(2.5, 2.0))
    cases["nearest_size_input"] = dict(n=1, c=5, in_hw=(10, 12), resize_type=1, ctm="NotSet", align=0, half=0, out_hw=(0, 0),
                                       size_input=(20, 30))
    cases["bilinear_op_scale"] = dict(n=2, c=3, in_hw=(9, 7), resize_type=2, ctm="NotSet", align=1, half=0, out_hw=(0, 0),
                                      scale_hw=(2.0, 3.0))
    cases["bilinear_nhwc"] = dict(n=1, c=6, in_hw=(8, 10), resize_type=2, ctm="PytorchHalfPixels", align=0, half=0,
                                  out_hw=(16, 20), nhwc=1)
    cases["cubic_nhwc"] = dict(n=2, c=5, in_hw=(7, 7), resize_type=3, ctm="AlignCorners", align=0, half=0, out_hw=(15, 13), nhwc=1)
    return cases


CASES = _cases()


def case_inputs(name):
    """x [n][c][ih][iw] float32 of a case"""
    c = CASES[name]
    seed = sorted(CASES).index(name) + 1000
    return np.random.default_rng(seed).standard_normal((c["n"], c["c"]) + tuple(c["in_hw"])).astype(np.float32) * 2


def case_out_hw(name):
    from oracle import interp_oracle as I
    c = CASES[name]
    if c.get("size_input"):
        return tuple(c["size_input"])
    return I.out_size(c["in_hw"], c["out_hw"], c.get("scale_hw", (0.0, 0.0)), c.get("scales"))


def case_transform(name):
    """(width_scale, height_scale, width_offset, height_offset) the geometry gives the lowered Interp of a case"""
    from oracle import interp_oracle as I
    c = CASES[name]
    return I.transform(c["resize_type"], c["ctm"], c["align"], c["half"], c["in_hw"], case_out_hw(name), c.get("scales"))


def case_oracle(name):
    """the restatement's output of a case"""
    from oracle import interp_oracle as I
    c = CASES[name]
    return I.interp(case_inputs(name), c["resize_type"], *case_transform(name), case_out_hw(name))


def case_reference(name, **kw):
    """the live reference's output of a case (refdump_interp op); kw: x2 / plugin as for interp_oracle.ref_interp"""
    from oracle import interp_oracle as I
    c = CASES[name]
    return I.ref_interp(case_inputs(name), c["resize_type"], c["ctm"], bool(c["align"]), bool(c["half"]), c["out_hw"],
                        c.get("scale_hw", (0.0, 0.0)), c.get("scales"), c.get("size_input"), bool(c.get("nhwc", 0)), **kw)


def digest(a):
    from oracle import llm_ops_oracle as L
    return L.digest(a)


def load():
    """{name: (shape, sha256)}"""
    z = np.load(PATH)
    return {name: (tuple(int(v) for v in z[f"{name}/shape"]), str(z[f"{name}/sha256"])) for name in CASES}


def main():
    sys.path.insert(0, ROOT)
    out = {}
    for name in CASES:
        y = case_reference(name)
        out[f"{name}/shape"] = np.array(y.shape, np.int64)
        out[f"{name}/sha256"] = np.array(digest(y))
        print(name, y.shape)
    np.savez_compressed(PATH, **out)
    print("wrote", PATH, os.path.getsize(PATH), "bytes")


if __name__ == "__main__":
    main()
