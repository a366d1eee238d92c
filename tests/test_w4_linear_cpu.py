"""4-bit LLM linear layers without a GPU: the oracle (mnn_oracle_linear_w4_dynamic_blocks) against the reference's recorded
outputs in tests/golden/w4_linear_golden.npz and against the live reference (skipped without oracle/_ref), and the GEMV and
GEMM kernels, which carry the 4-bit branches, compiled for sm_90a without register spills."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from mnn_b200 import build as B
from oracle import oracle as O
from oracle import w4_oracle as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "w4_linear_golden.npz")
# of max|y|.  Measured: at most 1.8e-6 over the 14 recorded cases (most outputs differ from the reference in the last bits:
# the reference's VNNI kernel associates the fp32 sums differently), the same order as the 8-bit blocked oracle's 4e-6
TOL = 4e-6
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
if not os.path.exists(NVCC):
    NVCC = shutil.which("nvcc") or NVCC


def cases():
    g = np.load(GOLD)
    for j in range(int(g["n"])):
        alpha, wmin, bias = g[f"c{j}_alpha"], g[f"c{j}_wmin"], g[f"c{j}_bias"]
        wz = (wmin - np.float32(-8) * alpha).astype(np.float32) if wmin.size else None
        yield j, g[f"c{j}_x"], g[f"c{j}_w"], alpha, wz, wmin, bias if bias.size else None, g[f"c{j}_y"]


def test_w4_golden_covers_the_issue_matrix():
    seen = set()
    for j, x, wp, alpha, wz, wmin, bias, y in cases():
        tokens, ic = x.shape
        oc, blocks = alpha.shape
        seen |= {("tokens", 1 if tokens == 1 else 8 if tokens <= 8 else 9), ("asym", wz is not None), ("bias", bias is not None),
                 ("bs", ic // blocks if blocks > 1 else 0), ("fast reorder", oc % 64 == 0)}
        assert wp.size * 2 == oc * ic and y.shape == (tokens, oc)
    for want in [("tokens", 1), ("tokens", 8), ("tokens", 9), ("asym", True), ("asym", False), ("bias", True), ("bias", False),
                 ("bs", 0), ("bs", 32), ("bs", 64), ("bs", 128), ("fast reorder", True), ("fast reorder", False)]:
        assert want in seen, want


def test_w4_oracle_matches_recorded_reference():
    worst = 0.0
    for j, x, wp, alpha, wz, _, bias, gold in cases():
        y = W.linear_w4_dynamic_blocks(x, wp, alpha.shape[0], alpha, wz, bias, alpha.shape[1])
        err = np.abs(y - gold).max() / np.abs(gold).max()
        assert err <= TOL, f"golden {j}: {err}"
        worst = max(worst, err)
    assert worst > 0.0      # the tolerance is used: the recording is not the oracle's own output


def test_w4_oracle_pack_and_unpack():
    """pack_w4 is load()'s layout (even index in the high nibble), and a 4-bit layer equals the 8-bit oracle on q + 8 with
    wzero - 8 alpha: the same real weights, so within fp32 rounding of each other"""
    rng = np.random.default_rng(8)
    q = rng.integers(-8, 8, (3, 6))
    wp = W.pack_w4(q)
    assert wp[0] == ((q[0, 0] + 8) << 4) | (q[0, 1] + 8)
    x = rng.uniform(-1, 1, (4, 128)).astype(np.float32)
    q = rng.integers(-8, 8, (24, 128)).astype(np.int8)
    alpha = rng.uniform(0.001, 0.01, (24, 2)).astype(np.float32)
    y4 = W.linear_w4_dynamic_blocks(x, W.pack_w4(q), 24, alpha, None, None, 2)
    y8 = O.linear_w8_dynamic_blocks(x, q, alpha, None, None, 2)
    assert np.abs(y4 - y8).max() <= 1e-5 * np.abs(y8).max()


def test_w4_oracle_against_live_reference():
    if not W.have_reference():
        pytest.skip("the reference core and its 4-bit harness (oracle/_ref) are not in this snapshot")
    for j, x, wp, alpha, wz, wmin, bias, gold in cases():
        if j % 3:
            continue
        oc, blocks = alpha.shape
        wire = np.stack([wmin, alpha], 2).ravel() if wz is not None else alpha.ravel()
        y = W.ref_linear(x, W.unpack_w4(wp, oc), wire, asym=wz is not None, bias=bias, blocks=blocks)
        assert np.array_equal(y, gold), f"golden {j}: the live reference no longer gives the recorded output"


@pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not found")
@pytest.mark.parametrize("src", ["linear_w8_gemv.cu", "gemm_i8_wgmma.cu"])
def test_w4_kernels_compile_without_spills(tmp_path, src):
    cmd = [NVCC, "-c", "-o", str(tmp_path / "k.o"), os.path.join(B.CSRC, src)] + B.NVCC_FLAGS + \
          B.PER_FILE_FLAGS.get(src, []) + ["-Xptxas", "-v"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    log = r.stdout + r.stderr
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(spills) >= (10 if "gemv" in src else 3), log[-2000:]
    assert all(s == ("0", "0") for s in spills), log[-3000:]


def test_w4_entry_is_declared():
    from mnn_b200 import _capi
    h = open(os.path.join(ROOT, "include", "mnn_b200.h")).read()
    assert "mnnb200_linear_w4_create_blocked(" in h
    assert "mnnb200_linear_w4_create_blocked" in _capi.SIGNATURES
