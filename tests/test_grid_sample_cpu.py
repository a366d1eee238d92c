"""The fp32 GridSample restatement (oracle/grid_sample_oracle.py) against the reference CPU: every recorded golden bit for bit, the
live reference where it is built (which pins the FMA finding: the unfused form differs), the float64 form within a rounding
bound, the exact fma32 helper on double-rounding cases; and the GridSample kernels compile without spills (CPU)."""
import os
import re
import subprocess

import numpy as np
import pytest

from oracle import grid_sample_oracle as S
from tests.golden import make_grid_sample_golden as G


@pytest.mark.parametrize("name", list(G.CASES))
def test_oracle_matches_golden(name):
    shape, sha = G.load()[name]
    y = G.case_oracle(name)
    assert y.shape == shape and y.dtype == np.float32
    assert G.digest(y) == sha


def test_golden_covers_the_forms():
    seen = {(c["rank"], c["mode"], c["padding"], c["align"]) for c in G.CASES.values()}
    assert seen == {(r, m, p, a) for r in (4, 5) for m in G.MODES for p in G.PADDINGS for a in (False, True)}
    shapes = [(c["n"], c["c"], c["in_dims"], c["out_dims"]) for c in G.CASES.values()]
    assert any(n > 1 for n, *_ in shapes) and all(c % 16 for _, c, *_ in shapes)
    for cmp in (lambda i, o: o[-1] > i[-1], lambda i, o: o[-1] < i[-1], lambda i, o: o == i):
        assert any(cmp(i, o) for *_, i, o in shapes)
    sp = np.array(G.SPECIALS, np.float32)
    assert np.isnan(sp).any() and np.isposinf(sp).any() and np.isneginf(sp).any() and (np.abs(sp) == 1e10).sum() == 2
    assert any(np.signbit(v) and v == 0 for v in sp)


@pytest.mark.parametrize("name", [n for n in G.CASES if "bilinear" in n])
def test_unfused_form_differs_from_the_golden(name):
    """the AVX2 (unfused) sequence does not reproduce the recorded AVX-512 CPU: the contraction is part of the parity target"""
    assert G.digest(G.case_oracle(name, fused=False)) != G.load()[name][1]


@pytest.mark.parametrize("name", list(G.CASES))
def test_float64_form_bounds_the_restatement(name):
    c = G.CASES[name]
    x, g = G.case_inputs(name)
    y = G.case_oracle(name)
    y64 = S.grid_sample64(x, g, c["mode"], c["padding"], c["align"])
    tame = (np.abs(g) <= 1.5).all(-1)[:, None]          # pixels of ordinary coordinates: weights in [0, 1]
    tame = np.broadcast_to(tame, y.shape)
    if c["mode"] == "nearest":
        assert np.array_equal(y[tame], y64[tame])
    else:   # taps^2 products and sums: a few ulp of the taps' magnitude
        assert np.abs(y[tame] - y64[tame]).max() <= 1e-5 * np.abs(x).max()


@pytest.mark.parametrize("name", list(G.CASES))
def test_oracle_matches_live_reference(name):
    if not S.have_refdump():
        pytest.skip("oracle/_ref/refdump_grid_sample is built by build() where the reference sources are")
    y = G.case_reference(name)
    assert np.array_equal(y.view(np.uint32), G.case_oracle(name, fused=S.host_fused()).view(np.uint32))


@pytest.mark.parametrize("rank", [4, 5])
def test_linear_input_is_read_as_packed(rank):
    """an x handed to the CPU op in NCHW instead of NC4HW4 is read (and y written) as if packed: the live reference equals
    grid_sample_linear_misread with the host's pack, not the sampling of the tensors as their format says"""
    if not S.have_refdump():
        pytest.skip("oracle/_ref/refdump_grid_sample is built by build() where the reference sources are")
    pack = 16 if S.host_fused() else 8
    rng = np.random.default_rng(rank)
    xs, gs = ((2, 32, 7, 9), (2, 5, 6, 2)) if rank == 4 else ((2, 16, 4, 5, 6), (2, 3, 4, 5, 3))
    x = rng.standard_normal(xs).astype(np.float32)
    g = rng.uniform(-1.1, 1.1, gs).astype(np.float32)
    for mode in ("bilinear", "nearest"):
        y = S.ref_grid_sample(x, g, mode, "border", False, linear_x=True)
        want = S.grid_sample_linear_misread(x, g, mode, "border", False, pack=pack, fused=S.host_fused())
        assert np.array_equal(y.view(np.uint32), want.view(np.uint32)), mode
        assert not np.array_equal(y, S.grid_sample(x, g, mode, "border", False))


def _fma_exact(a, b, c):
    """a * b + c rounded once to float32 (nearest, ties to even), from the exact rational value"""
    from fractions import Fraction
    v = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    f = np.float32(float(v))
    cands = [np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))]
    return min(cands, key=lambda q: (abs(Fraction(float(q)) - v), int(q.view(np.uint32)) & 1))


def test_fma32_exact_on_double_rounding_cases():
    """cases where the float64 sum a * b + c lands exactly on a float32 tie and rounding it again would round the wrong way"""
    f = np.float32
    one_ulp = f(2.0 ** -23)
    cases = [
        # a * b = 1 + 2^-24 + 2^-48 exactly; float64 keeps it, plain float32 rounding of the float64 value is correct here
        (f(1 + 2.0 ** -23), f(1 + 2.0 ** -23), f(0)),
        # product 1 + 2^-11 + 2^-24 (a float32 tie) plus a tiny c: the true sum is off the tie, float64 loses c and the tie
        # then rounds to even, the wrong way for a positive c
        (f(1 + 2.0 ** -12), f(1 + 2.0 ** -12), f(2.0 ** -60)),
        (f(1 + 2.0 ** -12), f(1 + 2.0 ** -12), f(-2.0 ** -60)),
        (f(3), f(1 + 2.0 ** -22), f(-2.0 ** -70)),
        (f(-1.5), f(1 + one_ulp), f(1e-30)),
    ]
    for a, b, c in cases:
        want = _fma_exact(a, b, c)
        got = S.fma32(a, b, c)
        assert got.view(np.uint32) == np.float32(want).view(np.uint32), (a, b, c, got, want)
    # the second case: naive float64 then float32 rounds to the even neighbour below, the exact fma one ulp above
    a, b, c = cases[1]
    naive = np.float32(np.float64(a) * np.float64(b) + np.float64(c))
    assert naive != S.fma32(a, b, c)
    # specials: NaN, infinities and signed zeros as IEEE fma gives them
    assert np.isnan(S.fma32(f(np.inf), f(0), f(1)))
    assert S.fma32(f(-0.0), f(1), f(-0.0)).view(np.uint32) == f(-0.0).view(np.uint32)
    assert S.fma32(f(-0.0), f(1), f(0.0)).view(np.uint32) == f(0.0).view(np.uint32)


def test_grid_sample_kernel_compiles_without_spills(tmp_path):
    from mnn_b200 import build as B
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    src = "grid_sample_f32.cu"
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
    names = [n for n in found if "grid_sample_f32_kernel" in n]
    assert len(names) == 8, found
    assert all(found[n] == 0 for n in names), {n: found[n] for n in names}
