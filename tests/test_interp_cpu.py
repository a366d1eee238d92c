"""The fp32 Interp restatement (oracle/interp_oracle.py) against the reference CPU: every recorded golden bit for bit, the live
reference where it is built, the float64 form within a rounding bound; and the Interp kernel compiles without spills (CPU)."""
import os
import re
import subprocess

import numpy as np
import pytest

from oracle import interp_oracle as I
from tests.golden import make_interp_golden as G


@pytest.mark.parametrize("name", list(G.CASES))
def test_oracle_matches_golden(name):
    shape, sha = G.load()[name]
    y = G.case_oracle(name)
    assert y.shape == shape and y.dtype == np.float32
    assert G.digest(y) == sha


def test_golden_covers_the_forms():
    seen = {(c["resize_type"], f) for n, c in G.CASES.items() for f in G.FORMS if n.endswith("_" + f)}
    assert seen == {(t, f) for t in G.TYPES for f in G.FORMS}
    shapes = [(c["n"], c["c"], c["in_hw"], G.case_out_hw(n)) for n, c in G.CASES.items()]
    assert any(o[1] % 4 for *_, o in shapes) and any(n > 1 for n, *_ in shapes) and any(c % 4 for _, c, *_ in shapes)
    assert any(i == (1, 1) for *_, i, _ in shapes) and any(o == (1, 1) for *_, o in shapes)
    assert any(o[0] < i[0] for *_, i, o in shapes) and any(o[0] % i[0] for *_, i, o in shapes)
    for key in ("scales", "size_input", "scale_hw", "nhwc"):
        assert any(key in c for c in G.CASES.values()), key


@pytest.mark.parametrize("name", list(G.CASES))
def test_float64_form_bounds_the_restatement(name):
    c = G.CASES[name]
    x = G.case_inputs(name)
    y, y64 = G.case_oracle(name), I.interp64(x, c["resize_type"], *G.case_transform(name), G.case_out_hw(name))
    if c["resize_type"] in (1, 4):
        assert np.array_equal(y, y64)
    else:   # taps^2 products and sums, weights rounded to float: a few ulp of the taps' magnitude
        assert np.abs(y - y64).max() <= 1e-5 * max(np.abs(x).max(), 1.0)


@pytest.mark.parametrize("name", ["bilinear_pytorch", "cubic_half", "round_tfhalf", "bilinear_scales_input", "cubic_nhwc"])
def test_oracle_matches_live_reference(name):
    if not I.have_refdump():
        pytest.skip("oracle/_ref/refdump_interp is built by build() where the reference sources are")
    y = G.case_reference(name)
    assert np.array_equal(y.view(np.uint32), G.case_oracle(name).view(np.uint32))


def test_cubic_taps_of_a_negative_coordinate_follow_truncation():
    """half-pixel at the top / left edge: the taps start at (int)src - 1 (truncation toward zero) while the fraction is
    src - floor(src), one tap off a textbook cubic, as the CPU computes it"""
    ws, hs, wo, ho = I.transform(3, "HalfPixels", 0, 0, (4, 4), (8, 8))
    idx, w = I.axis_table(3, ws, wo, 4, 8)
    assert wo < 0 and idx[0].tolist() == [0, 0, 1, 2]
    assert np.isclose(w[0].sum(), 1.0, atol=1e-6)


def test_interp_kernel_compiles_without_spills(tmp_path):
    from mnn_b200 import build as B
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    src = "interp_f32.cu"
    cmd = [nvcc, "-c", os.path.join(B.CSRC, src), "-o", str(tmp_path / "k.o")] + B.NVCC_FLAGS + B.PER_FILE_FLAGS[src] + \
          ["-Xptxas", "-v"]
    out = subprocess.run(cmd, capture_output=True, text=True, check=True).stderr
    found, fn = {}, None
    for line in out.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            fn = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and fn:
            found[fn] = int(m.group(1)) + int(m.group(2))
    names = [n for n in found if "interp_f32_kernel" in n]
    assert len(names) == 6, found
    assert all(found[n] == 0 for n in names), {n: found[n] for n in names}
