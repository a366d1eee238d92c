"""CPU tests of the fp32 Deconvolution's float64 oracle (oracle/deconv_oracle.py) against outputs recorded from the reference CPU
backend (tests/golden/deconv_f32_golden.npz) and, where oracle/_ref holds the harness, against the live reference; and that the
new kernels compile for sm_90a without spills."""
import os
import re
import subprocess

import numpy as np
import pytest

from oracle import deconv_oracle as D
from tests.golden import make_deconv_golden as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def golden_check(y, name, golden, tol):
    """y (full output) against the recorded outputs of case `name` within tol * max|recorded|"""
    rec, idx, shape = golden[name]
    assert tuple(y.shape) == shape, (y.shape, shape)
    flat = np.asarray(y, np.float64).reshape(-1)
    got = flat if idx is None else flat[idx]
    err = float(np.abs(got - rec).max() / max(np.abs(rec).max(), 1e-30))
    assert err <= tol, f"{name}: rel err {err:.2e} against the reference CPU"
    return err


def oracle_for(name, shape):
    n, ic, oc, hw, k, s, pads, d, op, same, out, dw, relu, relu6 = G.CASES[name]
    x, w, b = G.case_inputs(name)
    y, _ = D.deconv_f32(x, w, b, s, G.begin_pads(name, shape[2:]), d, 2 if relu6 else relu, out_hw=shape[2:], depthwise=bool(dw))
    return y


@pytest.mark.parametrize("name", list(G.CASES))
def test_oracle_matches_golden(name):
    golden = G.load()
    golden_check(oracle_for(name, golden[name][2]), name, golden, 1e-5)


def test_golden_covers_the_forms():
    golden = G.load()
    assert len(golden) == len(G.CASES) >= 12
    # a 1x1 stride-2 layer has phases without taps: whole output rows that are the bias alone
    _, idx, shape = golden["k1_s2"]
    assert idx is None and shape[2] == 2 * (G.CASES["k1_s2"][3][0] - 1) + 1


# (stride, pads [t, l, b, r], dilation, out_pads, same, output shape, depthwise, relu, relu6), fresh inputs
LIVE = [(2, (1, 1, 1, 1), 1, (0, 0), 0, None, 0, 1, 0), (3, (0, 2, 1, 0), 2, (1, 2), 0, None, 0, 0, 1),
        (2, (0, 0, 0, 0), 1, (0, 0), 1, (11, 9), 0, 0, 0), (2, (1, 0, 1, 0), 1, (1, 0), 0, None, 1, 0, 0)]


@pytest.mark.parametrize("case", range(len(LIVE)))
def test_oracle_matches_live_reference(case):
    if not D.have_refdump():
        pytest.skip("oracle/_ref/refdump_deconv is built by build() where the reference sources are")
    s, pads, d, op, same, out, dw, relu, relu6 = LIVE[case]
    rng = np.random.default_rng(40 + case)
    ic, oc, k = 6, 6 if dw else 5, 3
    x = rng.standard_normal((2, ic, 6, 5)).astype(np.float32)
    w = rng.standard_normal((ic, k, k) if dw else (ic, oc, k, k)).astype(np.float32) * 0.3
    b = rng.standard_normal(oc).astype(np.float32)
    y = D.ref_deconv(x, w, b, s, pads, d, op, bool(same), out, bool(dw), bool(relu), bool(relu6))
    pt, pl = pads[:2]
    if same:
        pt, pl = ((6 - 1) * s + k - y.shape[2]) // 2, ((5 - 1) * s + k - y.shape[3]) // 2
    ref, _ = D.deconv_f32(x, w, b, s, (pt, pl), d, 2 if relu6 else relu, out_hw=y.shape[2:], depthwise=bool(dw))
    assert np.abs(y - ref).max() <= 1e-5 * np.abs(ref).max()


def test_deconv_kernels_compile_without_spills(tmp_path):
    src, kernels = "deconv_f32_wgmma.cu", ("deconv_f32_wgmma_kernel", "pack_deconv_w_f32_kernel", "dwdeconv_f32_kernel")
    from mnn_b200 import build as B
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc, "-c", os.path.join(B.CSRC, src), "-o", str(tmp_path / "k.o")] + B.NVCC_FLAGS + ["-Xptxas", "-v"]
    out = subprocess.run(cmd, capture_output=True, text=True, check=True).stderr
    found, fn = {}, None
    for line in out.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            fn = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and fn:
            found[fn] = int(m.group(1)) + int(m.group(2))
    for k in kernels:
        names = [n for n in found if k in n]
        assert names, f"{k} not compiled"
        assert all(found[n] == 0 for n in names), {n: found[n] for n in names}
