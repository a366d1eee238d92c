"""The conv-group kernel (conv_group_wgmma.cu) as ptxas compiles it for sm_90a, checked without a GPU: no register spills in
any tile-width instantiation, and every column run of the epilogue is branch-free.  A column run is the requant chains of
one tile's column pairs for both accumulator rows of a thread, each chain ending in an F2I.TRUNC; with a branch region around
every pair the chains execute one after another, and the epilogue dominates the kernel's time."""
import os
import re
import shutil
import subprocess

import pytest

from mnn_b200 import build as B

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
if not os.path.exists(NVCC):
    NVCC = shutil.which("nvcc") or NVCC
CUOBJDUMP = os.path.join(os.path.dirname(NVCC), "cuobjdump")
SRC = os.path.join(B.CSRC, "conv_group_wgmma.cu")

pytestmark = pytest.mark.skipif(not (os.path.exists(NVCC) and os.path.exists(CUOBJDUMP)), reason="nvcc / cuobjdump not found")

CONTROL = ("BSSY", "BSYNC", "BRA", "BRX", "JMP", "JMX", "CALL", "RET", "EXIT", "BREAK", "WARPSYNC")


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    cubin = str(tmp_path_factory.mktemp("conv_group") / "conv_group_wgmma.cubin")
    cmd = [NVCC, "-cubin", "-o", cubin, SRC] + B.NVCC_FLAGS + B.PER_FILE_FLAGS.get(os.path.basename(SRC), []) + ["-Xptxas", "-v"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    sass = subprocess.run([CUOBJDUMP, "-sass", cubin], capture_output=True, text=True, check=True).stdout
    return r.stdout + r.stderr, sass


def kernel_instructions(sass):
    """the instructions of conv_group_wgmma_kernel, predicate guards stripped"""
    parts = re.split(r"^\s*Function : (\S+)", sass, flags=re.M)
    bodies = [body for name, body in zip(parts[1::2], parts[2::2]) if "conv_group_wgmma_kernel" in name]
    assert len(bodies) == 1
    out = []
    for ins in re.findall(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", bodies[0]):
        toks = [t for t in ins.split() if not t.startswith("@")]
        out.append(toks[0])
    return out


def test_no_spills(compiled):
    ptxas, _ = compiled
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", ptxas)
    assert spills, ptxas
    assert all(s == "0" and l == "0" for s, l in spills), ptxas


def test_epilogue_column_runs_are_branch_free(compiled):
    # split the kernel at every control-flow instruction and count the F2I.TRUNCs of each branch-free stretch: a whole column
    # run is 2 rows x bn / 8 column pairs x 2 outputs (bn = 16 ... 128), so a stretch holds 8 ... 64 of them, a multiple of 8
    _, sass = compiled
    counts, cur = [], 0
    for op in kernel_instructions(sass):
        if op.startswith(CONTROL):
            if cur:
                counts.append(cur)
            cur = 0
        elif op.startswith("F2I.TRUNC"):
            cur += 1
    if cur:
        counts.append(cur)
    assert counts, "no F2I.TRUNC in the kernel"
    bad = sorted(set(c for c in counts if c % 8 or not 8 <= c <= 64))
    assert not bad, f"branch-free stretches with {bad} F2I.TRUNC: an epilogue column run is split by control flow"
    # every tile width (16 ... 128) has its own runs
    assert set(range(8, 65, 8)) <= set(counts), sorted(set(counts))
