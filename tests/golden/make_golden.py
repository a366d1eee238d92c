"""Generates tests/golden/*.npz by running the UNMODIFIED reference CPU backend (oracle/_ref/refdump,
built from /root/reference by oracle/build_ref.py).  Run in the build container:  python tests/golden/make_golden.py
The fixtures are committed so the GPU box (no /root/reference, possibly no oracle/_ref) still has real-reference vectors.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import oracle as O  # noqa: E402
from tests.cases import KAT_SWEEP, kat_conv, random_modern_case  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def conv_golden():
    out = {}
    i = 0
    for case in KAT_SWEEP:
        (ic, oc), (kh, kw), n, pad, stride, dilate, (ih, iw) = case
        x, w, bias, scale = kat_conv(n, ic, ih, iw, oc, kh, kw)
        y = O.ref_conv(0, x, w, bias, scale, stride=stride, pad=pad, dilate=dilate)
        out.update({f"c{i}_mode": 0, f"c{i}_x": x, f"c{i}_w": w, f"c{i}_bias": bias, f"c{i}_scale": scale,
                    f"c{i}_stride": stride, f"c{i}_pad": pad, f"c{i}_dilate": dilate, f"c{i}_y": y,
                    f"c{i}_relu": 0, f"c{i}_s_in": 0.0, f"c{i}_s_out": 0.0, f"c{i}_z_in": 0, f"c{i}_z_out": 0})
        i += 1
    rng = np.random.default_rng(2024)
    for (ic, oc, kh, kw, n, ih, iw, st, pad, relu, dl) in [
            (3, 32, 3, 3, 2, 16, 16, (2, 2), (1, 1), 1, (1, 1)),      # MobileNet-v2 stem shape class
            (32, 16, 1, 1, 2, 14, 14, (1, 1), (0, 0), 0, (1, 1)),     # pointwise projection (no relu)
            (16, 96, 1, 1, 1, 14, 14, (1, 1), (0, 0), 1, (1, 1)),     # pointwise expansion
            (96, 24, 1, 1, 3, 7, 7, (1, 1), (0, 0), 0, (1, 1)),
            (160, 40, 1, 1, 2, 7, 7, (1, 1), (0, 0), 1, (1, 1)),      # ragged oc (not a multiple of 16)
            (24, 20, 3, 3, 1, 9, 11, (1, 1), (1, 1), 1, (2, 2)),      # dilation + pad with non-zero zero point
            (64, 64, 3, 3, 1, 8, 8, (1, 1), (1, 1), 1, (1, 1)),       # ResNet 3x3 class
            (20, 10, 7, 1, 2, 12, 5, (2, 1), (3, 0), 0, (1, 1))]:     # asymmetric kernel
        c = random_modern_case(rng, ic, oc, kh, kw, n, ih, iw, st, pad, relu, dl)
        y = O.ref_conv(1, c["x"], c["w"], c["bias"], c["ws"], stride=st, pad=pad, dilate=dl, relu=relu,
                       z_in=c["z_in"], z_out=c["z_out"], scale_in=c["s_in"], scale_out=c["s_out"])
        out.update({f"c{i}_mode": 1, f"c{i}_x": c["x"], f"c{i}_w": c["w"], f"c{i}_bias": c["bias"],
                    f"c{i}_scale": c["ws"], f"c{i}_stride": st, f"c{i}_pad": pad, f"c{i}_dilate": dl, f"c{i}_y": y,
                    f"c{i}_relu": relu, f"c{i}_s_in": c["s_in"], f"c{i}_s_out": c["s_out"], f"c{i}_z_in": c["z_in"],
                    f"c{i}_z_out": c["z_out"]})
        i += 1
    out["ncase"] = i
    np.savez_compressed(os.path.join(HERE, "conv_int8_golden.npz"), **out)
    print("conv_int8_golden.npz:", i, "cases")



def dw_linear_golden():
    """depthwise int8 conv + dynamic-quant linear outputs from the real reference (refdump conv mode 1 / linear)."""
    rng = np.random.default_rng(77)
    out = {}
    i = 0
    for (ch, k, n, ih, iw, st, pad, relu) in [(32, 3, 2, 16, 16, (1, 1), (1, 1), 1), (96, 3, 1, 15, 15, (2, 2), (1, 1), 1),
                                              (40, 5, 1, 9, 11, (1, 1), (2, 2), 0), (7, 3, 3, 6, 6, (1, 1), (0, 0), 1)]:
        x = rng.integers(-128, 128, (n, ch, ih, iw)).astype(np.int8)
        w = rng.integers(-127, 128, (ch, 1, k, k)).astype(np.int8)
        s_in, s_out = 0.043, 0.061
        z_in, z_out = int(rng.integers(-4, 5)), int(rng.integers(-4, 5))
        ws = (rng.uniform(0.003, 0.012, ch) / k * s_out / s_in).astype(np.float32)
        bias = (rng.uniform(-1, 1, ch) * 10 * s_out).astype(np.float32)
        y = O.ref_conv(1, x, w, bias, ws, stride=st, pad=pad, group=ch, relu=relu, z_in=z_in, z_out=z_out,
                       scale_in=s_in, scale_out=s_out)
        out.update({f"d{i}_x": x, f"d{i}_w": w, f"d{i}_ws": ws, f"d{i}_bias": bias, f"d{i}_stride": st, f"d{i}_pad": pad,
                    f"d{i}_relu": relu, f"d{i}_q": np.array([s_in, z_in, s_out, z_out], np.float64), f"d{i}_y": y})
        i += 1
    out["ndw"] = i
    j = 0
    # the last five: ONE token = the decode step, where the reference switches to its single-quant arithmetic (asymmetric input
    # quantisation over the row incl. the pack padding, zero point folded into the bias; ConvInt8TiledExecutor.cpp:1033, 1432, 2016-2050)
    for (tokens, ic, oc, asym, hb, lo, hi) in [(8, 64, 48, False, True, -1, 1), (33, 256, 200, True, True, -1, 1),
                                               (5, 96, 33, False, False, -1, 1), (64, 512, 128, True, False, -1, 1),
                                               (1, 2048, 512, True, True, -1, 1), (1, 100, 64, False, False, 0.2, 1.0),
                                               (1, 250, 33, True, False, -1, -0.1), (1, 320, 200, True, True, -3, 5),
                                               (1, 64, 48, False, True, 0.25, 0.25)]:
        x = rng.uniform(lo, hi, (tokens, ic)).astype(np.float32)
        wq = rng.integers(-128, 128, (oc, ic)).astype(np.int8)
        alpha = rng.uniform(0.001, 0.01, oc).astype(np.float32)
        wmin = rng.uniform(-0.05, 0.05, oc).astype(np.float32) if asym else np.zeros(0, np.float32)
        bias = rng.uniform(-1, 1, oc).astype(np.float32) if hb else np.zeros(0, np.float32)
        al = np.stack([wmin, alpha], 1).ravel() if asym else alpha
        y = O.ref_linear(x, wq, al, asym=asym, bias=bias if hb else None)
        out.update({f"l{j}_x": x, f"l{j}_wq": wq, f"l{j}_alpha": alpha, f"l{j}_wmin": wmin, f"l{j}_bias": bias, f"l{j}_y": y})
        j += 1
    out["nlin"] = j
    np.savez_compressed(os.path.join(HERE, "dw_linear_golden.npz"), **out)
    print("dw_linear_golden.npz:", i, "depthwise,", j, "linear cases")


def block_linear_golden():
    """K-blocked weight scales (MNN-LLM's default export, quant_block 64 / 128) through the real reference: prefill (>= 2 tokens)
    and decode (1 token) cases.  Oracle-only for now: the CUDA path declines block-wise layers (DESIGN.md section 9)."""
    rng = np.random.default_rng(78)
    out = {}
    j = 0
    for (tokens, ic, oc, blocks, asym, hb, lo, hi) in [(4, 256, 64, 4, False, False, -1, 1), (9, 512, 96, 8, True, True, -1, 1),
                                                       (33, 384, 40, 3, True, False, -1, 1), (1, 256, 64, 2, False, True, -1, 1),
                                                       (1, 512, 96, 4, True, True, 0.1, 2.0), (1, 128, 33, 2, True, False, -2, -0.5)]:
        x = rng.uniform(lo, hi, (tokens, ic)).astype(np.float32)
        wq = rng.integers(-128, 128, (oc, ic)).astype(np.int8)
        alpha = rng.uniform(0.001, 0.01, (oc, blocks)).astype(np.float32)
        wmin = rng.uniform(-0.05, 0.05, (oc, blocks)).astype(np.float32) if asym else np.zeros(0, np.float32)
        bias = rng.uniform(-1, 1, oc).astype(np.float32) if hb else np.zeros(0, np.float32)
        al = np.stack([wmin, alpha], 2).ravel() if asym else alpha.ravel()
        y = O.ref_linear(x, wq, al, asym=asym, bias=bias if hb else None, blocks=blocks)
        out.update({f"b{j}_x": x, f"b{j}_wq": wq, f"b{j}_alpha": alpha, f"b{j}_wmin": wmin, f"b{j}_bias": bias, f"b{j}_y": y})
        j += 1
    out["n"] = j
    np.savez_compressed(os.path.join(HERE, "block_linear_golden.npz"), **out)
    print("block_linear_golden.npz:", j, "cases")


def model_weight_hashes():
    """sha256 of every conv's weights/alpha as decoded BY THE REFERENCE (ConvolutionCommon::load via `refdump export`)."""
    import hashlib
    import json
    import tempfile
    model = os.path.join(HERE, "mbv2_int8.mnn")
    out = {}
    with tempfile.TemporaryDirectory() as d:
        O._run_refdump(["export", model, d])
        for line in open(os.path.join(d, "convs.txt")):
            name, opname, wsize, asize, asym = line.strip().split("|")
            idx = int(name.split("_")[1])
            w = open(os.path.join(d, name + ".w8"), "rb").read()
            a = open(os.path.join(d, name + ".alpha"), "rb").read()
            out[str(idx)] = dict(op=opname, w=hashlib.sha256(w).hexdigest(), alpha=hashlib.sha256(a).hexdigest(),
                                 n=int(wsize))
    json.dump(out, open(os.path.join(HERE, "mbv2_int8_weights_sha256.json"), "w"), indent=0)
    print("mbv2_int8_weights_sha256.json:", len(out), "convs")



def model_checkpoints():
    """Per-op outputs of the REAL reference on tests/golden/mbv2_int8.mnn (batch 1, seed 7): a subset is committed
    (the full per-op comparison runs live against oracle/_ref/refdump where it is present)."""
    import tempfile
    model = os.path.join(HERE, "mbv2_int8.mnn")
    keep = ["MobilenetV2/Conv/Conv2D", "MobilenetV2/expanded_conv/depthwise/depthwise", "MobilenetV2/expanded_conv/project/Conv2D",
            "MobilenetV2/expanded_conv_2/add", "MobilenetV2/expanded_conv_6/project/Conv2D", "MobilenetV2/expanded_conv_13/depthwise/depthwise",
            "MobilenetV2/expanded_conv_16/project/Conv2D", "MobilenetV2/Conv_1/Conv2D", "MobilenetV2/Logits/AvgPool",
            "MobilenetV2/Logits/Conv2d_1c_1x1/Conv2D", "MobilenetV2/Predictions/Softmax"]
    out = {}
    with tempfile.TemporaryDirectory() as d:
        recs = O.ref_run_model(model, 1, 7, d, 1)
        out["input"] = np.fromfile(os.path.join(d, "input.f32"), np.float32).reshape(1, 3, 224, 224)
        names = []
        for r in recs:
            if r["name"] in keep and r["scale"] > 0:
                f = np.fromfile(os.path.join(d, r["file"]), np.float32).reshape(r["dims"])
                q = np.rint(f / np.float32(r["scale"]) + np.float32(r["zero"])).astype(np.int8)
                out[f"t{len(names)}"] = q
                names.append(r["name"])
        last = recs[-1]
        out["output"] = np.fromfile(os.path.join(d, last["file"]), np.float32).reshape(last["dims"])
    out["names"] = np.array(names)
    np.savez_compressed(os.path.join(HERE, "mbv2_int8_checkpoints.npz"), **out)
    print("mbv2_int8_checkpoints.npz:", len(names), "tensors")



def wino_golden():
    """int8 Winograd conv outputs from the real reference, AVX2 build (oracle/_ref/refdump_avx2 wino): the reference
    test's own generator (test/op/ConvInt8Test.cpp:566-600) at F(2,3) plus calibrated random cases at F(2/4/6,3)."""
    from tests.cases import kat_wino, random_wino_case, wino_oracle
    assert O.have_reference_avx2(), "python oracle/build_ref.py --avx2"
    rng = np.random.default_rng(4242)
    cases = [(2, kat_wino(2, 32, 32, 39, 47))]
    for (unit, n, ic, oc, ih, iw, pad, relu) in [(2, 2, 16, 24, 12, 15, 1, True), (2, 1, 40, 33, 9, 7, 0, False),
                                                 (4, 2, 32, 16, 14, 14, 1, True), (4, 1, 13, 21, 11, 18, 1, False),
                                                 (6, 1, 32, 32, 19, 15, 1, True), (6, 2, 8, 20, 7, 9, 0, False)]:
        cases.append((unit, random_wino_case(rng, unit, n, ic, oc, ih, iw, pad, relu)))
    out = {"ncase": len(cases)}
    for i, (unit, c) in enumerate(cases):
        y = wino_oracle(O, c, unit, O.ref_wino)
        out[f"w{i}_unit"] = unit
        out[f"w{i}_y"] = y
        for k, v in c.items():
            out[f"w{i}_{k}"] = np.asarray(v)
    np.savez_compressed(os.path.join(HERE, "wino_int8_golden.npz"), **out)
    print("wino_int8_golden.npz:", len(cases), "cases")



def matmul_golden():
    """float MatMul / BatchMatMul outputs of the real reference CPU backend (refdump matmul)."""
    from tests.test_matmul import CASES, make
    rng = np.random.default_rng(808)
    out = {"ncase": len(CASES)}
    for i, (bd, e, l, h, ta, tb) in enumerate(CASES):
        a, b = make(rng, bd, e, l, h, ta, tb)
        out.update({f"m{i}_a": a, f"m{i}_b": b, f"m{i}_ta": ta, f"m{i}_tb": tb, f"m{i}_y": O.ref_matmul(a, b, ta, tb)})
    np.savez_compressed(os.path.join(HERE, "matmul_golden.npz"), **out)
    print("matmul_golden.npz:", len(CASES), "cases")


def pool_golden():
    """float Pooling outputs of the real reference CPU backend (refdump poolf): AVE on every config of tests/test_pool.py, MAX
    on the ones whose windows start past the input or lie wholly in the padding."""
    from tests.test_pool import POOL_CONFIGS, pool_input, pool_kwargs
    rng = np.random.default_rng(909)
    out = {}
    cases = [(ci, True) for ci in range(len(POOL_CONFIGS))] + [(3, False), (14, False), (18, False)]
    for i, (ci, is_avg) in enumerate(cases):
        x = pool_input(rng, 2, 3, POOL_CONFIGS[ci])
        out.update({f"p{i}_cfg": ci, f"p{i}_avg": int(is_avg), f"p{i}_x": x,
                    f"p{i}_y": O.ref_pool_f32(x, is_avg, **pool_kwargs(POOL_CONFIGS[ci]))})
    out["ncase"] = len(cases)
    np.savez_compressed(os.path.join(HERE, "pool_golden.npz"), **out)
    print("pool_golden.npz:", len(cases), "cases")


if __name__ == "__main__":
    # python tests/golden/make_golden.py [conv] [dw_linear] [block_linear] [hashes] [checkpoints] [wino] [matmul] [pool]
    # (default: all)
    assert O.have_reference(), "build oracle/_ref first: python oracle/build_ref.py"
    which = set(sys.argv[1:]) or {"conv", "dw_linear", "block_linear", "hashes", "checkpoints", "wino", "matmul", "pool"}
    if "conv" in which:
        conv_golden()
    if "dw_linear" in which:
        dw_linear_golden()
    if "block_linear" in which:
        block_linear_golden()
    if "hashes" in which:
        model_weight_hashes()
    if "checkpoints" in which:
        model_checkpoints()
    if "wino" in which:
        wino_golden()
    if "matmul" in which:
        matmul_golden()
    if "pool" in which:
        pool_golden()
