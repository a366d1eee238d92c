"""Parity AT THE BENCH CONFIGS THEMSELVES (-m gpu): the sizes BASELINE.json's configs name -- not smaller stand-ins -- checked
against the reference's outputs recorded by tests/golden/make_config_golden.py (hashes of the bit-exact outputs, sampled rows of
the fp32 ones); the plugin legs need the reference core itself (oracle/_ref) and run only where it was built.

  C2  MobileNet-v2 int8 .mnn, batch 32: every command's int8 output, plugin vs MNN_FORWARD_CPU and WholeNetSession vs
      MNN_FORWARD_CPU (position-weighted 64-bit sums of the dequantised tensors: REFDUMP_HASH=1, oracle/refdump.cpp)
  C3  ResNet-50 3x3/s1 layers at batch 64 on int8 Winograd F(6,3): C=64/56x56 and C=512/7x7 vs the AVX2 reference build
  C4  Qwen-1.8B linear shapes at 4096 tokens: 2048->6144 (+bias, asymmetric) and 5504->2048 vs `refdump linear`
  +   a .mnn whose Convolution carries a winogradAttr through the PLUGIN (reference AVX2 core + libmnn_b200_plugin.so)
"""
import hashlib
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import oracle as O
from tests.golden.make_config_golden import C4_CASES, c3_case, c4_inputs

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLUGIN = os.path.join(ROOT, "mnn_b200", "libmnn_b200_plugin.so")
MODEL = os.path.join(ROOT, "tests", "golden", "mbv2_int8.mnn")
GOLDEN = os.path.join(ROOT, "tests", "golden", "config_golden.npz")
FP_INTERNAL = ("MobilenetV2/Predictions/Softmax",)      # expf vs the reference's polynomial: +-1 LSB (documented in DESIGN.md)
needs_ref2 = pytest.mark.skipif(not O.have_reference_avx2(), reason="oracle/_ref/refdump_avx2 not on this box")


def wsum64(a: np.ndarray) -> int:
    """the hash refdump prints under REFDUMP_HASH=1: sum_k word[k] * (k * 0x9E3779B97F4A7C15 + 1) mod 2^64 over the fp32 words"""
    w = np.ascontiguousarray(a, np.float32).view(np.uint32).ravel().astype(np.uint64)
    k = np.arange(w.size, dtype=np.uint64)
    with np.errstate(over="ignore"):
        return int((w * (k * np.uint64(0x9E3779B97F4A7C15) + np.uint64(1))).sum(dtype=np.uint64))


def _refdump_run(exe, libdir, model, batch, seed, outdir, threads, plugin, hash_only=True):
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = libdir + ":" + os.path.join(ROOT, "mnn_b200") + ":" + env.get("LD_LIBRARY_PATH", "")
    env["REFDUMP_HASH"] = "1" if hash_only else "0"
    if plugin:
        env["REFDUMP_PLUGIN"] = PLUGIN
    else:
        env.pop("REFDUMP_PLUGIN", None)
    os.makedirs(outdir, exist_ok=True)
    r = subprocess.run([exe, "run", model, str(batch), str(seed), outdir, str(threads)], env=env, capture_output=True, text=True,
                       timeout=1800)
    assert r.returncode == 0, r.stderr[-2000:] + r.stdout[-500:]
    recs = []
    for line in open(os.path.join(outdir, "index.txt")):
        f, name, typ, dims, qs, qz, qmin, qmax, aq = line.rstrip("\n").split("|")
        recs.append(dict(file=f, name=name, type=typ.strip(), dims=[int(v) for v in dims.split(",")] if dims else [],
                         scale=float(qs), zero=float(qz), apply_quant=int(aq)))
    stats = [json.loads(l) for l in r.stdout.splitlines() if l.startswith("{\"plugin_")]
    return recs, (stats[-1] if stats else None)


def _diagnose(d, batch, threads, ncmd):
    """a hash mismatch says nothing about how many values differ: re-run both sides up to the failing command with full dumps"""
    os.environ["REFDUMP_MAX_COMMANDS"] = str(ncmd)
    try:
        cpu, _ = _refdump_run(O.REFDUMP, O.REF_DIR, MODEL, batch, 5, os.path.join(d, "dcpu"), threads, False, hash_only=False)
        gpu, _ = _refdump_run(O.REFDUMP, O.REF_DIR, MODEL, batch, 5, os.path.join(d, "dgpu"), 4, True, hash_only=False)
    finally:
        os.environ.pop("REFDUMP_MAX_COMMANDS", None)
    a = np.fromfile(os.path.join(d, "dcpu", cpu[ncmd - 1]["file"]), np.float32)
    b = np.fromfile(os.path.join(d, "dgpu", gpu[ncmd - 1]["file"]), np.float32)
    xa = np.fromfile(os.path.join(d, "dcpu", "input.f32"), np.float32)
    xb = np.fromfile(os.path.join(d, "dgpu", "input.f32"), np.float32)
    bad = np.flatnonzero(a != b)
    signed_zero = int(np.count_nonzero((a == b) & (np.signbit(a) != np.signbit(b))))
    return (f"inputs equal: {np.array_equal(xa, xb)}; {bad.size} of {a.size} values differ (first at {bad[:5].tolist()}, "
            f"cpu {a[bad[:5]].tolist()} vs plugin {b[bad[:5]].tolist()}), max |diff| {np.abs(a - b).max() if bad.size else 0}; "
            f"{signed_zero} equal values with different zero sign")


def test_c2_mbv2_batch32_every_op_plugin_and_session_vs_cpu_backend():
    """BASELINE configs[1] at its own batch: the WholeNetSession host against MNN_FORWARD_CPU on refdump's 32 x 3 x 224 x 224
    seed-5 input (the recorded position-weighted 64-bit sums of the dequantised tensors, REFDUMP_HASH=1), every int8 tensor
    bit-exact (softmax +-1 LSB excluded); where the reference core is built, also the unmodified reference pipeline on the plugin
    against MNN_FORWARD_CPU in the same run."""
    from mnn_b200.session import WholeNetSession
    batch = 32
    g = np.load(GOLDEN)
    cpu = [dict(name=str(n), file=str(h), scale=float(sc), zero=float(z), dims=[int(v) for v in str(dm).split(",")])
           for n, h, sc, z, dm in zip(g["b32_names"], g["b32_hash"], g["b32_scale"], g["b32_zero"], g["b32_dims"])]
    if O.have_reference():
        assert os.path.exists(PLUGIN), "mnn_b200/libmnn_b200_plugin.so is missing although the reference core is present"
        threads = min(os.cpu_count() or 1, 32)
        with tempfile.TemporaryDirectory() as d:
            live, _ = _refdump_run(O.REFDUMP, O.REF_DIR, MODEL, batch, 5, os.path.join(d, "cpu"), threads, False)
            gpu, stats = _refdump_run(O.REFDUMP, O.REF_DIR, MODEL, batch, 5, os.path.join(d, "gpu"), 4, True)
            assert stats is not None and stats["plugin_declined"] == 0, stats
            assert [(r["name"], r["type"]) for r in live] == [(r["name"], r["type"]) for r in gpu]
            n_int8 = 0
            for idx, (a, b) in enumerate(zip(live, gpu)):
                if a["apply_quant"] and a["name"] not in FP_INTERNAL:
                    if a["file"] != b["file"]:
                        raise AssertionError(f"plugin vs CPU backend differ at batch 32: {a['name']} ({a['type']}): " +
                                             _diagnose(d, batch, threads, idx + 1))
                    n_int8 += 1
            assert n_int8 >= 60, n_int8
    # the C-ABI host on the same input
    x = O.refdump_input(5, (batch, 3, 224, 224))
    sess = WholeNetSession(MODEL, batch)
    sess.capture()
    sess.set_input(x)
    sess.run()
    checked = 0
    for r in cpu:
        if r["name"] not in sess.checkpoints or r["name"] in FP_INTERNAL:
            continue
        q = sess.read_int8(r["name"]).reshape(r["dims"])
        f = (q.astype(np.float32) - np.float32(r["zero"])) * np.float32(r["scale"])       # MNNInt8ScaleToFloat
        assert r["file"] == "hash:%016x" % wsum64(f), f"WholeNetSession vs CPU backend differ at batch 32: {r['name']}"
        checked += 1
    assert checked >= 60, checked


@pytest.mark.parametrize("C_,HW", [(64, 56), (512, 7)])
def test_c3_resnet_f63_batch64_vs_live_reference(backend, C_, HW):
    """BASELINE configs[2]: ResNet-50 3x3/s1, batch 64, int8 Winograd F(6,3) -- the first and the last layer class, full size,
    bit-exact against the reference's AVX2 build (ConvInt8Winograd; its output's sha256 is recorded)."""
    from tests.test_winograd import run_wino
    y, ex = run_wino(backend, c3_case(C_, HW), 6)
    assert y.shape == (64, C_, HW, HW)
    assert hashlib.sha256(np.ascontiguousarray(y).tobytes()).hexdigest() == str(np.load(GOLDEN)[f"c3_{C_}_{HW}"]), \
        "F(6,3) output differs from the reference's"
    assert (np.abs(y.astype(int)) == 127).mean() < 0.5
    assert ex.cost()[1] == 64.0 * HW * HW * C_ * C_ * 9


@pytest.mark.parametrize("ic,oc,asym,has_bias", C4_CASES)
def test_c4_qwen_linear_4096_tokens_vs_live_reference(backend, ic, oc, asym, has_bias):
    """BASELINE configs[3]: the two extreme Qwen-1.8B linear shapes at the full 4096 tokens against the reference CPU backend's
    dynamic-quant W8A8 (`refdump linear`, Memory_Low; sampled rows and max|y| recorded), 1e-3 relative (north_star); both
    product kernels (single CTA / CTA pair)."""
    from mnn_b200.backend import Op, Tensor
    import torch
    T = 4096
    x, wq, alpha, wmin, bias = c4_inputs(ic, oc, asym, has_bias)
    g = np.load(os.path.join(ROOT, "tests", "golden", f"config_c4_{ic}_{oc}.npz"))
    rows, ref, absmax = g["rows"], g["y"], float(g["absmax"])
    # refdump is fed the wire form {min, scale}; the C ABI takes the offset of SIGNED int8 weights (see _signed_offset)
    from mnn_b200 import _capi
    for variant in (2, 3):
        op = Op(type="LinearW8", conv=dict(ic=ic, oc=oc), weight=wq, wscale=alpha,
                wzero=None if wmin is None else _signed_offset(wmin, alpha), bias=bias)
        xt = Tensor((T, ic), "float", None, torch.from_numpy(x).cuda())
        yt = Tensor((T, oc), "float", None, torch.full((T, oc), float("nan"), dtype=torch.float32, device="cuda"))
        ex = backend.onCreate([xt], [yt], op)
        _capi.check(_capi.lib().mnnb200_conv_int8_set_variant(ex._h, variant))
        assert ex.onResize([xt], [yt]) == 0
        assert ex.onExecute([xt], [yt]) == 0
        backend.onSync()
        y = yt.data.cpu().numpy()
        assert np.isfinite(y).all(), f"variant {variant}: unwritten outputs"
        assert abs(np.abs(y).max() - absmax) <= 1e-3 * absmax, f"variant {variant}: max|y| {np.abs(y).max()} vs {absmax}"
        err = np.abs(y[rows] - ref).max() / absmax
        assert err <= 1e-3, f"variant {variant}: rel err {err}"


def _signed_offset(wmin, alpha):
    """ConvolutionCommon::load turns the wire 'min' into the offset of SIGNED int8 weights: min - clampMin * scale with
    clampMin = -128 (source/core/ConvolutionCommon.cpp:757-766)."""
    return (wmin - np.float32(-128.0) * alpha).astype(np.float32)


@needs_ref2
def test_winograd_attr_mnn_through_the_plugin():
    """INTEGRATION.md gap of round 1: a converted .mnn whose Convolution carries a winogradAttr, scheduled by the UNMODIFIED
    reference core (AVX2 build, the one whose ConvInt8Winograd is right) on MNN_FORWARD_CUDA = the plugin, equals the same
    process's MNN_FORWARD_CPU result bit for bit, with nothing declined."""
    assert os.path.exists(PLUGIN)
    model = os.path.join(ROOT, "tests", "golden", "wino_modern_conv.mnn")
    with tempfile.TemporaryDirectory() as d:
        cpu, _ = _refdump_run(O.REFDUMP_AVX2, O.REF_DIR, model, 2, 9, os.path.join(d, "cpu"), 1, False, hash_only=False)
        gpu, stats = _refdump_run(O.REFDUMP_AVX2, O.REF_DIR, model, 2, 9, os.path.join(d, "gpu"), 1, True, hash_only=False)
        assert stats is not None and stats["plugin_declined"] == 0 and stats["plugin_created"] >= 1, stats
        assert [(r["name"], r["type"]) for r in cpu] == [(r["name"], r["type"]) for r in gpu]
        convs = 0
        for a, b in zip(cpu, gpu):
            fa = np.fromfile(os.path.join(d, "cpu", a["file"]), np.float32)
            fb = np.fromfile(os.path.join(d, "gpu", b["file"]), np.float32)
            if a["apply_quant"]:
                assert np.array_equal(fa, fb), f"{a['name']} ({a['type']}): {np.count_nonzero(fa != fb)} of {fa.size} differ"
                convs += "Convolution" in a["type"]
            else:
                assert np.abs(fa - fb).max() <= 1e-3 * max(np.abs(fa).max(), 1e-12)
        assert convs >= 1
