"""Writes tests/golden/rnn_golden.npz: ONNX LSTM / RNN outputs (Y, Y_h[, Y_c]) recorded from the reference CPU backend
(oracle/_ref/refdump_rnn op, built by build() where the reference sources are).

Each case's inputs are rebuilt from its seed by `case_inputs` (numpy's PCG64 generator, the same on every machine).  The
comparison is by tolerance (the CPU's sigmoid and tanh are clamped polynomials), so outputs are stored as float32.  An LSTM
with h0 but no c0 has no golden: the reference CPU crashes on it (tests/test_rnn_cpu.py pins that).
Run: python tests/golden/make_rnn_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
PATH = os.path.join(ROOT, "tests", "golden", "rnn_golden.npz")

# name -> (cell 0 LSTM / 1 RNN, T, B, I, H, D, init 'none' | 'h0' | 'h0c0', weight scale (None: 1 / sqrt(H)))
CASES = {
    "lstm_d1_none": (0, 5, 3, 7, 6, 1, "none", None),
    "lstm_d1_states_b_ne_h": (0, 6, 3, 20, 33, 1, "h0c0", None),
    "lstm_d2_none": (0, 4, 2, 9, 5, 2, "none", None),
    "lstm_d2_states": (0, 5, 4, 6, 3, 2, "h0c0", None),
    "lstm_b1": (0, 4, 1, 8, 33, 1, "h0c0", None),
    "lstm_t1": (0, 1, 5, 4, 7, 2, "h0c0", None),
    "lstm_h1": (0, 3, 2, 5, 1, 1, "h0c0", None),
    "lstm_saturated": (0, 4, 3, 10, 9, 2, "h0c0", 6.0),
    "rnn_d1_none": (1, 5, 3, 7, 6, 1, "none", None),
    "rnn_d1_h0_b_ne_h": (1, 6, 3, 20, 33, 1, "h0", None),
    "rnn_d2_h0": (1, 4, 2, 9, 3, 2, "h0", None),
    "rnn_d2_none_t1": (1, 1, 4, 5, 5, 2, "none", None),
    "rnn_h1_b1": (1, 3, 1, 4, 1, 1, "h0", None),
    "rnn_saturated": (1, 4, 3, 10, 9, 2, "h0", 6.0),
}


def case_inputs(name):
    """(cell, x, w, r, b, h0, c0) of a case, from its seed"""
    cell, T, B, I, H, D, init, scale = CASES[name]
    rng = np.random.default_rng(sorted(CASES).index(name) + 700)
    G = 4 if cell == 0 else 1
    s = scale if scale is not None else 1.0 / np.sqrt(H)
    x = rng.standard_normal((T, B, I)).astype(np.float32)
    w = (rng.standard_normal((D, G * H, I)) * s).astype(np.float32)
    r = (rng.standard_normal((D, G * H, H)) * s).astype(np.float32)
    b = (rng.standard_normal((D, G * H)) * 0.5).astype(np.float32)
    h0 = (rng.standard_normal((D, B, H)) * 0.5).astype(np.float32) if init != "none" else None
    c0 = rng.standard_normal((D, B, H)).astype(np.float32) if init == "h0c0" else None
    return cell, x, w, r, b, h0, c0


def main():
    sys.path.insert(0, ROOT)
    from oracle import rnn_oracle as R
    out = {}
    for name in sorted(CASES):
        cell, x, w, r, b, h0, c0 = case_inputs(name)
        for k, y in zip(("y", "y_h", "y_c"), R.ref_op(cell, x, w, r, b, h0, c0)):
            out[f"{name}/{k}"] = y.astype(np.float32)
    np.savez_compressed(PATH, **out)
    print(f"wrote {PATH}: {len(CASES)} cases, {os.path.getsize(PATH)} bytes")


if __name__ == "__main__":
    main()
