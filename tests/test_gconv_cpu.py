"""CPU tests of the grouped fp32 Convolution: the float64 restatement (oracle/gconv_oracle.py) against outputs recorded from the
reference CPU backend (tests/golden/gconv_f32_golden.npz) and, where oracle/_ref holds the harness, against the live reference;
the grouped kernel's n-chunk mapping and block-diagonal weight packing, restated in numpy, against the grouped conv; and that the
conv kernel compiles for sm_90a without spills."""
import os
import re
import subprocess

import numpy as np
import pytest

from oracle import gconv_oracle as D
from tests.golden import make_gconv_golden as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def golden_check(y, name, golden, tol):
    """y (full output) against the recorded outputs of case `name` within tol * max|recorded|: the relative error"""
    rec, idx, shape = golden[name]
    assert tuple(y.shape) == shape, (y.shape, shape)
    flat = np.asarray(y, np.float64).reshape(-1)
    got = flat if idx is None else flat[idx]
    err = float(np.abs(got - rec).max() / max(np.abs(rec).max(), 1e-30))
    assert err <= tol, f"{name}: rel err {err:.2e} against the reference CPU"
    return err


def oracle_for(name):
    n, ic, oc, hw, k, s, pads, d, group, input_count, relu, relu6 = G.CASES[name]
    x, w, b = G.case_inputs(name)
    y, _ = D.gconv_f32(x, w, b, D.cpu_group(group, input_count, ic), s, pads, d, 2 if relu6 else relu)
    return y


# The CPU runs the 5x5 stride-1 groups of the AlexNet case as Winograd (ConvolutionFloatFactory: bestWinogradUnit), whose
# transforms cost it 3.2e-4 of max|y| against float64; every other case is a direct fp32 GEMM, within 2.5e-6.
CPU_WINOGRAD = {"alexnet_g2_k5": 5e-4}


@pytest.mark.parametrize("name", list(G.CASES))
def test_oracle_matches_golden(name):
    err = golden_check(oracle_for(name), name, G.load(), CPU_WINOGRAD.get(name, 1e-5))
    print(f"{name}: the reference CPU's fp32 output is within {err:.2e} of float64 (max|d| / max|y|)")


def test_golden_covers_the_forms():
    golden = G.load()
    assert len(golden) == len(G.CASES) >= 12
    groups = {name: (c[1] // c[8], c[2] // c[8]) for name, c in G.CASES.items()}       # (icg, ocg)
    assert groups["depth_multiplier2"] == (1, 2) and groups["ocg160_g2"][1] > 128
    assert G.CASES["inputcount_per_group"][9] * G.CASES["inputcount_per_group"][8] == G.CASES["inputcount_per_group"][1]
    assert any(c[5] != 1 for c in G.CASES.values()) and any(c[7] != 1 for c in G.CASES.values())


# (n, ic, oc, (ih, iw), k, stride, pads, dilation, group, inputCount, relu, relu6), fresh inputs: Express's and the TensorFlow
# inputCount, ReLU6, a group of one input channel, and one past the 128-wide tile
LIVE = [(2, 24, 48, (7, 6), 3, 1, (1, 1, 1, 1), 1, 3, 24, 1, 0), (2, 24, 48, (7, 6), 3, 2, (0, 1, 1, 0), 1, 3, 8, 0, 1),
        (1, 12, 24, (6, 5), 3, 1, (2, 2, 2, 2), 2, 12, 12, 0, 0), (1, 10, 300, (4, 4), 1, 1, (0, 0, 0, 0), 1, 2, 10, 1, 0)]


@pytest.mark.parametrize("case", range(len(LIVE)))
def test_oracle_matches_live_reference(case):
    if not D.have_refdump():
        pytest.skip("oracle/_ref/refdump_gconv is built by build() where the reference sources are")
    n, ic, oc, hw, k, s, pads, d, group, input_count, relu, relu6 = LIVE[case]
    rng = np.random.default_rng(70 + case)
    x = rng.standard_normal((n, ic) + hw).astype(np.float32)
    w = (rng.standard_normal((oc, ic // group, k, k)) * 0.3).astype(np.float32)
    b = rng.standard_normal(oc).astype(np.float32)
    y = D.ref_gconv(x, w, b, group, input_count, s, pads, d, bool(relu), bool(relu6))
    ref, _ = D.gconv_f32(x, w, b, D.cpu_group(group, input_count, ic), s, pads, d, 2 if relu6 else relu)
    assert y.shape == ref.shape
    assert np.abs(y - ref).max() <= 1e-5 * np.abs(ref).max()


def chunk_plan(G_, icg, ocg):
    """capi.cu conv_f32_create for group > 1: (bn, P, Q, n_chunks, cp8)"""
    bn = 32 if ocg <= 32 else 64 if ocg <= 64 else 128
    P = min(bn // ocg, G_) if ocg <= bn else 1
    Q = 1 if ocg <= bn else -(-ocg // bn)
    n_chunks = -(-G_ // P) if Q == 1 else G_ * Q
    return bn, P, Q, n_chunks, -(-P * icg // 8) * 8


def chunked_conv(x, w, b, G_, stride, pads):
    """the grouped kernel's arithmetic in float64: per n chunk, the loader's input channels, pack_conv_w_f32_kernel's block-diagonal
    weight rows (K = taps x cp8, channel-minor) and the epilogue's column -> channel map"""
    n, ic, ih, iw = x.shape
    oc, icg, kh, kw = w.shape
    ocg = oc // G_
    bn, P, Q, n_chunks, cp8 = chunk_plan(G_, icg, ocg)
    (pt, pl, pb, pr), (sh, sw) = pads, (stride, stride)
    oh, ow = D.out_size(ih, kh, sh, pt, pb, 1), D.out_size(iw, kw, sw, pl, pr, 1)
    xp = np.pad(x.astype(np.float64), ((0, 0), (0, 0), (pt, pb), (pl, pr)))
    y = np.full((n, oc, oh, ow), np.nan)
    taps = kh * kw
    for nc in range(n_chunks):
        g0, sub = nc // Q * P, nc % Q
        ng = min(P, G_ - g0)
        ic0, cin = g0 * icg, ng * icg
        oc0, ncols = g0 * ocg + sub * bn, min(bn, ng * ocg - sub * bn)
        # A: [M][taps * cp8], zero past cin
        A = np.zeros((n, oh, ow, taps, cp8))
        for t in range(taps):
            r, c = divmod(t, kw)
            A[..., t, :cin] = xp[:, ic0:ic0 + cin, r:r + sh * oh:sh, c:c + sw * ow:sw].transpose(0, 2, 3, 1)
        # B: [bn][taps * cp8], pack_conv_w_f32_kernel's rows
        B = np.zeros((bn, taps, cp8))
        for j in range(bn):
            ch = oc0 + j
            if j >= ncols or ch >= oc:
                continue
            lo = (ch // ocg - g0) * icg
            B[j, :, lo:lo + icg] = w[ch].reshape(icg, taps).T
        acc = A.reshape(n, oh, ow, -1) @ B.reshape(bn, -1).T
        y[:, oc0:oc0 + ncols] = acc[..., :ncols].transpose(0, 3, 1, 2) + np.asarray(b, np.float64)[oc0:oc0 + ncols, None, None]
    return y


@pytest.mark.parametrize("name", list(G.CASES))
def test_chunk_mapping_restates_the_grouped_conv(name):
    """every output channel written exactly by one chunk, and the block-diagonal GEMM equal to the grouped conv in float64"""
    n, ic, oc, hw, k, s, pads, d, group, input_count, relu, relu6 = G.CASES[name]
    if d != 1 or isinstance(k, tuple) or isinstance(s, tuple):
        pytest.skip("the restatement takes square kernels, one stride and no dilation")
    x, w, b = G.case_inputs(name)
    x = x[:1]
    y = chunked_conv(x, w, b, group, s, pads)
    ref, _ = D.gconv_f32(x, w, b, group, s, pads, 1, 0)
    assert not np.isnan(y).any()
    assert np.allclose(y, ref, rtol=1e-12, atol=1e-12 * np.abs(ref).max())


@pytest.mark.parametrize("shape,plan", [((32, 4, 4), (32, 8, 1, 4, 32)), ((5, 1, 160), (128, 1, 2, 10, 8)),
                                        ((7, 3, 9), (32, 3, 1, 3, 16)), ((3, 80, 80), (128, 1, 1, 3, 80)),
                                        ((16, 1, 2), (32, 16, 1, 1, 16)), ((2, 48, 128), (128, 1, 1, 2, 48))])
def test_chunk_plan(shape, plan):
    """(G, icg, ocg) -> (bn, P, Q, n_chunks, cp8): whole groups per chunk up to the narrowest width that holds one, G not a
    multiple of P, and Q chunks per group past 128 output channels"""
    assert chunk_plan(*shape) == plan


def test_conv_kernel_compiles_without_spills(tmp_path):
    from mnn_b200 import build as B
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc, "-c", os.path.join(B.CSRC, "conv_f32_wgmma.cu"), "-o", str(tmp_path / "k.o")] + B.NVCC_FLAGS + ["-Xptxas", "-v"]
    out = subprocess.run(cmd, capture_output=True, text=True, check=True).stderr
    found, regs, fn = {}, {}, None
    for line in out.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            fn = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and fn:
            found[fn] = int(m.group(1)) + int(m.group(2))
        m = re.search(r"Used (\d+) registers", line)
        if m and fn:
            regs[fn] = int(m.group(1))
    for bn in (32, 64, 128):
        names = [f for f in found if "conv_f32_wgmma_kernelILi%dE" % bn in f]
        assert names and all(found[f] == 0 for f in names), {f: found[f] for f in names}
        print(f"conv_f32_wgmma_kernel<{bn}>: {regs[names[0]]} registers, no spills")
    names = [f for f in found if "pack_conv_w_f32_kernel" in f]
    assert names and all(found[f] == 0 for f in names)
