"""Writes tests/golden/gru_golden.npz: GRU outputs recorded from the reference CPU backend (oracle/_ref/refdump_gru op, built
by build() where the reference sources are).

Each case's inputs are rebuilt from its seed by `case_inputs` (numpy's PCG64 generator, the same on every machine).  The
comparison is by tolerance (the CPU's sigmoid and tanh are clamped polynomials), so outputs are stored as float32.  Y_h is not
stored where the reference CPU leaves its backward half unset (two directions, Y and Y_h both requested, and h0: the op's
scratch, oracle/gru_oracle.py cpu_y_h); without h0 that half is the scratch's zeros, and is stored as recorded.
Run: python tests/golden/make_gru_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
PATH = os.path.join(ROOT, "tests", "golden", "gru_golden.npz")

# name -> (linear_before_reset, T, B, I, H, D, h0, keepAllOutputs, outputs, weight scale (None: 1 / sqrt(H)))
CASES = {
    "lbr0_d1_none": (0, 5, 3, 7, 6, 1, False, True, 2, None),
    "lbr0_d1_h0_b_ne_h": (0, 6, 3, 20, 33, 1, True, True, 2, None),
    "lbr0_d2_none": (0, 4, 2, 9, 5, 2, False, True, 2, None),
    "lbr0_d2_h0_y_only": (0, 5, 4, 6, 3, 2, True, True, 1, None),
    "lbr0_d2_h0_t1_y_h_only": (0, 1, 5, 4, 7, 2, True, False, 1, None),
    "lbr0_b9_h17": (0, 3, 9, 5, 17, 1, True, True, 2, None),
    "lbr0_saturated": (0, 4, 3, 10, 9, 2, True, True, 1, 6.0),
    "lbr1_d1_none": (1, 5, 3, 7, 6, 1, False, True, 2, None),
    "lbr1_d1_h0_b_ne_h": (1, 6, 3, 20, 33, 1, True, True, 2, None),
    "lbr1_d2_none": (1, 4, 2, 9, 5, 2, False, True, 2, None),
    "lbr1_d2_h0_y_only": (1, 5, 4, 6, 3, 2, True, True, 1, None),
    "lbr1_d1_none_t1_y_h_only": (1, 1, 2, 3, 4, 1, False, False, 1, None),
    "lbr1_b11_h12": (1, 3, 11, 8, 12, 2, False, True, 2, None),
    "lbr1_saturated": (1, 4, 3, 10, 9, 1, True, True, 2, 6.0),
}


def case_inputs(name):
    """(lbr, keepAllOutputs, outputs, x, params, h0) of a case, from its seed"""
    lbr, T, B, I, H, D, hh, keep, n_out, scale = CASES[name]
    rng = np.random.default_rng(sorted(CASES).index(name) + 900)
    from oracle import gru_oracle as G
    x = rng.standard_normal((T, B, I)).astype(np.float32)
    params = G.random_params(rng, D, I, H, scale)
    h0 = (rng.standard_normal((D, B, H)) * 0.5).astype(np.float32) if hh else None
    return lbr, keep, n_out, x, params, h0


def main():
    sys.path.insert(0, ROOT)
    from oracle import gru_oracle as G
    out = {}
    for name in sorted(CASES):
        lbr, keep, n_out, x, params, h0 = case_inputs(name)
        got = G.ref_op(lbr, x, params, h0, keep_all=keep, n_out=n_out)
        names = ("y", "y_h")[:n_out] if keep else ("y_h",)
        for k, y in zip(names, got):
            if k == "y_h" and keep and y.shape[0] == 2 and h0 is not None:
                continue
            out[f"{name}/{k}"] = y.astype(np.float32)
    np.savez_compressed(PATH, **out)
    print(f"wrote {PATH}: {len(CASES)} cases, {os.path.getsize(PATH)} bytes")


if __name__ == "__main__":
    main()
