"""The Gather / GatherND / GatherElements / Cast restatement (oracle/gather_oracle.py) against the reference CPU: every recorded
golden bit for bit, the live reference where it is built (including GatherND's batch dims reading the first batch, and every
MatMul golden within 1e-5), the float64 broadcast MatMul within 1e-5 of the recorded CPU; and the gather kernels compile without
spills (CPU)."""
import os
import re
import subprocess

import numpy as np
import pytest

from oracle import gather_oracle as G
from tests.golden import make_gather_golden as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _need_ref():
    if not G.have_refdump():
        pytest.skip("oracle/_ref/refdump_gather is built by build() where the reference sources are")


@pytest.mark.parametrize("name", list(M.CASES))
def test_oracle_matches_golden(name):
    shape, sha = M.load()[0][name]
    y = M.case_oracle(name)
    assert y.shape == shape and M.digest(y) == sha


@pytest.mark.parametrize("name", list(M.MATMUL_CASES))
def test_float64_matmul_matches_golden(name):
    y = M.load()[1][name]
    ref = M.matmul_oracle(name)
    assert y.shape == ref.shape and np.abs(y - ref).max() <= 1e-5 * np.abs(ref).max()


def test_golden_covers_the_forms():
    kinds = {c["kind"] for c in M.CASES.values()}
    assert kinds == {"Gather", "GatherV2", "GatherND", "GatherElements", "Cast"}
    inside = set()
    for n, c in M.CASES.items():
        if c["kind"] in ("Gather", "GatherV2"):
            p = c["params"][0]
            ax = (c["axis"] or 0) % len(p)
            inside.add(int(np.prod(p[ax + 1:])))
    assert {1, 3, 768} <= inside
    nd = [c for c in M.CASES.values() if c["kind"] == "GatherND"]
    assert {c["axis"] or 0 for c in nd} == {0, 1}
    for name in M.CASES:
        c = M.CASES[name]
        if c["kind"] == "Cast":
            continue
        x = M.case_inputs(name)
        assert G.cpu_defined(c["kind"], *x, c["axis"] or 0), name
    outside = [n for n in M.CASES if M.CASES[n]["kind"] != "Cast" and
               (M.case_inputs(n)[1] < 0).any() and (M.case_inputs(n)[1] >= 0).any()]
    assert len(outside) >= 3, "negative and out-of-range indices"
    a = {M.MATMUL_CASES[n][1:3] for n in M.MATMUL_CASES}
    assert ((2, 16, 64), (64, 48)) in a and ((1, 4, 32, 16), (2, 4, 16, 32)) in a
    assert any(len(s) == 1 for sa, sb in a for s in (sa, sb))


@pytest.mark.parametrize("name", list(M.CASES))
def test_oracle_matches_live_reference(name):
    _need_ref()
    y = M.case_reference(name)
    assert M.digest(y) == M.load()[0][name][1]
    assert np.array_equal(y.view(np.uint32), np.ascontiguousarray(M.case_oracle(name)).view(np.uint32))


@pytest.mark.parametrize("name", list(M.MATMUL_CASES))
def test_matmul_golden_matches_live_reference(name):
    _need_ref()
    y, ref = M.case_reference(name), M.load()[1][name]
    assert y.shape == ref.shape and np.abs(y - ref).max() <= 1e-5 * np.abs(ref).max()


def test_gathernd_batch_dims_read_the_first_batch():
    """the CPU's GatherND over one batch dim: out[b, j] = params[0][tuple], not params[b][tuple]"""
    _need_ref()
    rng = np.random.default_rng(7)
    p = rng.standard_normal((3, 6, 4)).astype(np.float32)
    idx = rng.integers(0, 6, (3, 5, 1)).astype(np.int32)
    y = G.ref_op("GatherND", [p, idx], axis=1)
    assert np.array_equal(y, G.gather_nd(p, idx, 1))
    assert np.array_equal(y, np.stack([p[0][idx[b, :, 0]] for b in range(3)]))
    assert not np.array_equal(y, np.stack([p[b][idx[b, :, 0]] for b in range(3)]))


def test_cpu_reads_another_row_where_the_kernels_zero_fill():
    """the documented difference: an index past the axis whose offset lies inside the params reads a later row on the CPU"""
    _need_ref()
    p = np.arange(2 * 3 * 4, dtype=np.float32).reshape(2, 3, 4)
    idx = np.array([1, 3], np.int32)                     # 3 >= the axis length 3; offset 12 < 24
    y = G.ref_op("GatherV2", [p, idx], axis=1)
    assert not G.cpu_defined("GatherV2", p, idx, 1)
    assert np.array_equal(y[0, 1], p.reshape(-1)[12:16])   # batch 0 reads batch 1's first row
    assert np.array_equal(G.gather(p, idx, 1)[:, 1], np.zeros((2, 4), np.float32))


def test_gather_kernels_compile_without_spills():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    src = os.path.join(ROOT, "mnn_b200", "csrc", "gather.cu")
    r = subprocess.run([nvcc, "-c", src, "-o", os.devnull, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        "--expt-relaxed-constexpr", "-Xptxas", "-v"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    entries = re.findall(r"Compiling entry function '(\w+)'", r.stderr)
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(entries) == 5 and len(spills) == 5, r.stderr
    assert all(s == ("0", "0") for s in spills), r.stderr
