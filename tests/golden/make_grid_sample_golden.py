"""Writes tests/golden/grid_sample_golden.npz: fp32 GridSample outputs recorded from the reference CPU backend of an AVX-512 host
(oracle/_ref/refdump_grid_sample op, built by build() where the reference sources are).

Each case's input and grid are rebuilt from its seed by `case_inputs` (numpy's PCG64 generator, the same on every machine); every
grid carries the special values of SPECIALS at its first entries.  The outputs are bit-exact targets, so the file holds only their
shape and the sha256 of their fp32 bytes.
Run: python tests/golden/make_grid_sample_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
PATH = os.path.join(ROOT, "tests", "golden", "grid_sample_golden.npz")

MODES = ("bilinear", "nearest")
PADDINGS = ("zeros", "border", "reflection")
# (n, c, in spatial dims, out spatial dims): out larger than, smaller than and equal to in, batch 2, channel counts not a multiple
# of 16 (the AVX-512 CPU packs 16)
SHAPES4 = [(2, 19, (7, 9), (12, 15)), (1, 5, (16, 12), (6, 5)), (2, 33, (8, 8), (8, 8))]
SHAPES5 = [(2, 3, (5, 6, 7), (3, 8, 9)), (1, 17, (6, 5, 4), (2, 3, 3)), (2, 4, (4, 4, 4), (4, 4, 4))]
# grid values that pin the CPU's edge arithmetic: the borders and their neighbours, integral and half-integral coordinates of a
# 7- or 8-wide axis (in both alignCorners conventions), values just outside, huge, infinite, NaN and -0
SPECIALS = [1.0, -1.0, 0.0, -0.0, np.nextafter(np.float32(1), np.float32(2)), np.nextafter(np.float32(-1), np.float32(-2)),
            1e10, -1e10, np.inf, -np.inf, np.nan, 0.25, 0.5, -0.5, 1 / 3, 0.75, 2.0 / 7, 1.0 / 7, 1.5, -1.5, 3e9 / 2 ** 31]


def _cases():
    cases = {}
    for rank, shapes in ((4, SHAPES4), (5, SHAPES5)):
        i = 0
        for mode in MODES:
            for pad in PADDINGS:
                for align in (False, True):
                    n, c, ind, outd = shapes[i % len(shapes)]
                    cases[f"r{rank}_{mode}_{pad}_{'align' if align else 'noalign'}"] = dict(
                        rank=rank, n=n, c=c, in_dims=ind, out_dims=outd, mode=mode, padding=pad, align=align)
                    i += 1
    return cases


CASES = _cases()


def case_inputs(name):
    """(x [n][c][(id)][ih][iw], grid [n][(od)][oh][ow][rank - 2]) float32 of a case: a grid over [-1.1, 1.1] with the
    special values first (distinct per batch)"""
    c = CASES[name]
    rng = np.random.default_rng(sorted(CASES).index(name) + 3000)
    x = (rng.standard_normal((c["n"], c["c"]) + tuple(c["in_dims"])) * 2).astype(np.float32)
    g = rng.uniform(-1.1, 1.1, (c["n"],) + tuple(c["out_dims"]) + (c["rank"] - 2,)).astype(np.float32)
    flat = g.reshape(c["n"], -1)
    sp = np.array(SPECIALS, np.float32)
    flat[0, :sp.size] = sp
    if c["n"] > 1:
        flat[1, :sp.size] = sp[::-1]
    return x, flat.reshape(g.shape)


def case_oracle(name, **kw):
    """the restatement's output of a case (kw: fused, as for grid_sample_oracle.grid_sample)"""
    from oracle import grid_sample_oracle as S
    c = CASES[name]
    x, g = case_inputs(name)
    return S.grid_sample(x, g, c["mode"], c["padding"], c["align"], **kw)


def case_reference(name, **kw):
    """the live reference's output of a case (refdump_grid_sample op); kw: more / plugin as for grid_sample_oracle.ref_grid_sample"""
    from oracle import grid_sample_oracle as S
    c = CASES[name]
    x, g = case_inputs(name)
    return S.ref_grid_sample(x, g, c["mode"], c["padding"], c["align"], **kw)


def digest(a):
    from oracle import llm_ops_oracle as L
    return L.digest(a)


def load():
    """{name: (shape, sha256)}"""
    z = np.load(PATH)
    return {name: (tuple(int(v) for v in z[f"{name}/shape"]), str(z[f"{name}/sha256"])) for name in CASES}


def main():
    sys.path.insert(0, ROOT)
    from oracle import grid_sample_oracle as S
    assert S.host_fused(), "the goldens are the AVX-512 CPU's: record them on an AVX-512 host"
    out = {}
    for name in CASES:
        y = case_reference(name)
        out[f"{name}/shape"] = np.array(y.shape, np.int64)
        out[f"{name}/sha256"] = np.array(digest(y))
    np.savez_compressed(PATH, **out)
    print(f"wrote {PATH}: {len(CASES)} cases")


if __name__ == "__main__":
    main()
