"""The conv-group kernel's epilogue stores (conv_group_wgmma.cu), checked in the SASS ptxas makes for sm_90a without a GPU.  The
GEMM columns of a chunk are permuted so that a thread holds 8 consecutive output channels of each row per 32-column group
(4 in a 16-wide last group): the int8 outputs leave in 8-byte (4-byte) stores, a warp store covers whole 32-byte sectors,
and no 2-byte store is left.  The accumulators start at the per-column sums, so the epilogue adds no per-output integer."""
import re

from tests.test_conv_group_sass import CONTROL, compiled, kernel_instructions  # noqa: F401  (compiled: module fixture)


def column_runs(sass):
    """the branch-free stretches of the kernel that hold F2I.TRUNCs, as lists of opcodes"""
    runs, cur = [], []
    for op in kernel_instructions(sass):
        if op.startswith(CONTROL):
            if any(o.startswith("F2I.TRUNC") for o in cur):
                runs.append(cur)
            cur = []
        else:
            cur.append(op)
    if any(o.startswith("F2I.TRUNC") for o in cur):
        runs.append(cur)
    return runs


def test_no_two_byte_global_store(compiled):
    _, sass = compiled
    ops = kernel_instructions(sass)
    assert not [o for o in ops if re.match(r"STG\.E\.(U?16|S16|U8|S8)", o)], sorted(set(o for o in ops if o.startswith("STG")))


def test_one_store_per_8_outputs(compiled):
    # a run of bn columns x 2 rows: bn / 32 full groups (one STG.E.64 = 8 outputs each, per row) and, when bn % 32 == 16, one
    # 16-wide group (one STG.E = 4 outputs, per row).  A run may be split across stretches at the row setup, so count over
    # all runs: every F2I.TRUNC belongs to exactly one store's 8 (or 4) outputs.
    _, sass = compiled
    ops = kernel_instructions(sass)
    f2i = sum(o.startswith("F2I.TRUNC") for o in ops)
    st64 = sum(o == "STG.E.64" for o in ops)
    st32 = sum(o == "STG.E" for o in ops)
    assert f2i == 8 * st64 + 4 * st32, (f2i, st64, st32)
    assert st64 and st32, (st64, st32)


def test_mode0_instructions_per_output(compiled):
    # the bn = 128 runs without the border correction (no LDG): 64 outputs per thread.  The parent epilogue took 16
    # instructions per output (2-byte stores, per-output column sum and pad select)
    _, sass = compiled
    runs = [r for r in column_runs(sass) if sum(o.startswith("F2I.TRUNC") for o in r) == 64 and not any(o.startswith("LDG") for o in r)]
    assert len(runs) == 2, [len(r) for r in runs]    # requant_fast and requant_fast_small
    per_output = max(len(r) for r in runs) / 64
    assert per_output < 13, per_output
