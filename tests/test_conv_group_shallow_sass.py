"""The shallow conv-group kernel (conv_group_shallow_wgmma.cu) as ptxas compiles it for sm_90a, checked without a GPU: its four
112-register consumer warpgroups hold every tile width up to kGroupShallowMaxBN (kernels.h) without spills, ptxas keeps the
wgmmas asynchronous, and every epilogue column run is one branch-free stretch, as in the conv-group kernel."""
import os
import re
import subprocess

import pytest

from mnn_b200 import build as B
from tests.test_conv_group_sass import CONTROL, CUOBJDUMP, NVCC, pytestmark  # noqa: F401  (pytestmark: skip without nvcc)

SRC = os.path.join(B.CSRC, "conv_group_shallow_wgmma.cu")


def shallow_max_bn():
    m = re.search(r"constexpr int kGroupShallowMaxBN = (\d+);", open(os.path.join(B.CSRC, "kernels.h")).read())
    assert m, "kGroupShallowMaxBN not found in kernels.h"
    return int(m.group(1))


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    cubin = str(tmp_path_factory.mktemp("conv_group_shallow") / "conv_group_shallow_wgmma.cubin")
    cmd = [NVCC, "-cubin", "-o", cubin, SRC] + B.NVCC_FLAGS + B.PER_FILE_FLAGS.get(os.path.basename(SRC), []) + ["-Xptxas", "-v"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    sass = subprocess.run([CUOBJDUMP, "-sass", cubin], capture_output=True, text=True, check=True).stdout
    return r.stdout + r.stderr, sass


def kernel_ops(sass):
    parts = re.split(r"^\s*Function : (\S+)", sass, flags=re.M)
    bodies = [body for name, body in zip(parts[1::2], parts[2::2]) if "conv_group_shallow_wgmma_kernel" in name]
    assert len(bodies) == 1
    return [[t for t in ins.split() if not t.startswith("@")][0] for ins in re.findall(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", bodies[0])]


def test_no_spills(compiled):
    ptxas, _ = compiled
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", ptxas)
    assert spills, ptxas
    assert all(s == "0" and l == "0" for s, l in spills), ptxas


def test_no_wgmma_serialization(compiled):
    ptxas, _ = compiled
    assert "wgmma.mma_async instructions are serialized" not in ptxas, ptxas


def test_column_runs_are_branch_free(compiled):
    # a column run is 2 rows x bn / 8 column pairs x 2 outputs = bn / 2 F2I.TRUNC: every branch-free stretch holds a whole
    # number of them, and every width 16 ... kGroupShallowMaxBN has its run
    _, sass = compiled
    counts, cur = [], 0
    for op in kernel_ops(sass):
        if op.startswith(CONTROL):
            if cur:
                counts.append(cur)
            cur = 0
        elif op.startswith("F2I.TRUNC"):
            cur += 1
    if cur:
        counts.append(cur)
    top = shallow_max_bn() // 2
    bad = sorted(set(c for c in counts if c % 8 or not 8 <= c <= top))
    assert not bad, f"branch-free stretches with {bad} F2I.TRUNC: an epilogue column run is split by control flow"
    assert set(counts) == set(range(8, top + 1, 8)), sorted(set(counts))


def test_register_split_fits_the_launch(compiled):
    # setmaxnreg.inc only takes registers that setmaxnreg.dec gave back in the same CTA: one producer warpgroup and four
    # consumer warpgroups after the split may hold no more than the 5 warpgroups at the launch's register count
    ptxas, _ = compiled
    used = [int(n) for n in re.findall(r"Used (\d+) registers", ptxas)]
    assert len(used) == 1, ptxas
    src = open(SRC).read()
    m = re.search(r"constexpr int kProducerRegs = (\d+), kConsumerRegs = (\d+);", src)
    assert m, "register split not found in " + SRC
    producer, consumer = int(m.group(1)), int(m.group(2))
    assert producer + 4 * consumer <= 5 * used[0], (producer, consumer, used[0])
    assert consumer == 112
