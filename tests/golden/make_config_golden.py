"""Records what the bench-config GPU tests compare against, from the LIVE reference built under oracle/_ref (run where the
reference sources exist: python tests/golden/make_config_golden.py).  Inputs are regenerated from seeds by the tests
(oracle.refdump_input, numpy generators), so only the reference's answers are stored:

  config_golden.npz    whole MobileNet-v2 at batch 2 (seed 11): sha256 of every int8 checkpoint (the softmax output in full);
                       batch 32 (seed 5): refdump's REFDUMP_HASH=1 hash of every dequantised int8 command output;
                       ResNet-50 3x3 F(6,3) at batch 64: sha256 of the reference's int8 output
  config_c4_<ic>_<oc>.npz  Qwen linear layers at 4096 tokens: fixed sampled rows of the reference output + max|y| over all rows
"""
import hashlib
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import oracle as O  # noqa: E402
from tests.cases import random_wino_case, wino_oracle  # noqa: E402

GOLD = os.path.dirname(os.path.abspath(__file__))
MODEL = os.path.join(GOLD, "mbv2_int8.mnn")
FP_INTERNAL = ("MobilenetV2/Predictions/Softmax",)
C3_CASES = [(64, 56), (512, 7)]
C4_CASES = [(2048, 6144, True, True), (5504, 2048, True, False)]
C4_ROWS = {6144: 24, 2048: 64}


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def c4_inputs(ic, oc, asym, has_bias):
    rng = np.random.default_rng(ic + oc)
    T = 4096
    x = rng.uniform(-1, 1, (T, ic)).astype(np.float32)
    wq = rng.integers(-128, 128, (oc, ic), dtype=np.int8)
    alpha = rng.uniform(0.001, 0.01, oc).astype(np.float32)
    wmin = (alpha * rng.uniform(-8, 8, oc)).astype(np.float32) if asym else None
    bias = rng.uniform(-1, 1, oc).astype(np.float32) if has_bias else None
    return x, wq, alpha, wmin, bias


def c4_rows(oc):
    return np.sort(np.random.default_rng(oc).choice(4096, C4_ROWS[oc], replace=False))


def c3_case(C_, HW):
    return random_wino_case(np.random.default_rng(C_ + HW), 6, 64, C_, C_, HW, HW, 1, True)


def main():
    assert O.have_reference() and O.have_reference_avx2(), "build the reference first (__graft_entry__.build())"
    out = {}
    with tempfile.TemporaryDirectory() as d:
        recs = O.ref_run_model(MODEL, 2, 11, d, 8)
        assert np.array_equal(np.fromfile(os.path.join(d, "input.f32"), np.float32).reshape(2, 3, 224, 224),
                              O.refdump_input(11, (2, 3, 224, 224)))
        names, hashes, full = [], [], {}
        for r in recs:
            if r["scale"] <= 0 or not r["apply_quant"]:
                continue
            f = np.fromfile(os.path.join(d, r["file"]), np.float32).reshape(r["dims"])
            q = np.rint(f / np.float32(r["scale"]) + np.float32(r["zero"])).astype(np.int8)
            names.append(r["name"])
            hashes.append(sha(q))
            if r["name"] in FP_INTERNAL:
                full[r["name"]] = q
        out["b2_names"] = np.array(names)
        out["b2_sha256"] = np.array(hashes)
        for i, n in enumerate(FP_INTERNAL):
            out[f"b2_full{i}"] = full[n]
    with tempfile.TemporaryDirectory() as d:
        env = dict(os.environ, REFDUMP_HASH="1", LD_LIBRARY_PATH=O.REF_DIR + ":" + os.environ.get("LD_LIBRARY_PATH", ""))
        env.pop("REFDUMP_PLUGIN", None)
        subprocess.run([O.REFDUMP, "run", MODEL, "32", "5", d, str(min(os.cpu_count() or 1, 32))], env=env, check=True,
                       capture_output=True)
        assert np.array_equal(np.fromfile(os.path.join(d, "input.f32"), np.float32).reshape(32, 3, 224, 224),
                              O.refdump_input(5, (32, 3, 224, 224)))
        names, hashes, scale, zero, dims = [], [], [], [], []
        for line in open(os.path.join(d, "index.txt")):
            f, name, typ, dm, qs, qz, qmin, qmax, aq = line.rstrip("\n").split("|")
            if not int(aq) or float(qs) <= 0:
                continue
            names.append(name); hashes.append(f); scale.append(float(qs)); zero.append(float(qz))
            dims.append(",".join(dm.split(",")))
        out["b32_names"] = np.array(names)
        out["b32_hash"] = np.array(hashes)
        out["b32_scale"] = np.array(scale, np.float32)
        out["b32_zero"] = np.array(zero, np.float32)
        out["b32_dims"] = np.array(dims)
    for C_, HW in C3_CASES:
        out[f"c3_{C_}_{HW}"] = np.array(sha(wino_oracle(O, c3_case(C_, HW), 6, O.ref_wino)))
    np.savez(os.path.join(GOLD, "config_golden.npz"), **out)
    for ic, oc, asym, has_bias in C4_CASES:
        x, wq, alpha, wmin, bias = c4_inputs(ic, oc, asym, has_bias)
        al = np.stack([wmin, alpha], 1).astype(np.float32).ravel() if asym else alpha
        ref = O.ref_linear(x, wq, al, asym=asym, bias=bias, threads=min(os.cpu_count() or 1, 32))
        rows = c4_rows(oc)
        np.savez(os.path.join(GOLD, f"config_c4_{ic}_{oc}.npz"), rows=rows, y=ref[rows], absmax=np.float32(np.abs(ref).max()))


if __name__ == "__main__":
    main()
