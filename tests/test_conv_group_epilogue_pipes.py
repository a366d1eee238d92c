"""The conv-group kernel's epilogue column runs (conv_group_wgmma.cu) counted by pipe, in the SASS ptxas makes for sm_90a without a
GPU.  The requant clamps the rounded integers: two F2I results are packed into a saturated s16 pair (I2IP), clamped with one
s16x2 min and one max (VIMNMX) and the low bytes of two pairs taken by one PRMT, so no float min / max (FMNMX) is left; the
+-0.5 is one LOP3; widths up to kConstRegsMaxBN hold a run's constants in registers, so their runs have no LDS."""
import re

from tests.test_conv_group_sass import SRC, compiled  # noqa: F401  (compiled: module fixture)
from tests.test_conv_group_stores import column_runs

# the instruction classes of a column run, by the pipe that executes them
PIPES = {
    "fp32": ("FADD", "FMUL", "FFMA"),
    "alu": ("LOP3", "PRMT", "FMNMX", "IMNMX", "VIMNMX", "I2IP", "ISETP", "SEL", "SHF", "IADD3", "VIADD", "LEA"),
    "conversion": ("F2I", "I2F", "I2FP"),
    "lds": ("LDS",),
    "store": ("STG",),
}


def outputs(run):
    return sum(o.startswith("F2I.TRUNC") for o in run)


def per_pipe(run):
    """instructions per output of a column run, by class; `other` is what no class names (IMAD, MOV, S2R, ...)"""
    n = outputs(run)
    split = {k: sum(o.split(".")[0] in ops for o in run) / n for k, ops in PIPES.items()}
    split["other"] = len(run) / n - sum(split.values())
    return split


def mode0_runs(sass, width):
    """the column runs of tile width `width` without the border correction (no LDG): width / 2 outputs per thread, small-K
    (int -> float on the FP32 pipe, no I2FP) or not"""
    return [r for r in column_runs(sass) if outputs(r) == width // 2 and not any(o.startswith("LDG") for o in r)]


def const_regs_max_bn():
    m = re.search(r"constexpr int kConstRegsMaxBN = (\d+);", open(SRC).read())
    assert m, "kConstRegsMaxBN not found in " + SRC
    return int(m.group(1))


def test_mode0_instructions_per_output_bn128(compiled):
    # the parent epilogue took 12.9 instructions per output here (two FMNMX per output, the +-0.5 in two LOP3s, bytes packed
    # by three PRMTs per 4 outputs, the pad mask built per tile)
    _, sass = compiled
    runs = mode0_runs(sass, 128)
    assert len(runs) == 2, [len(r) for r in runs]
    assert max(len(r) for r in runs) / 64 < 10.5, [len(r) / 64 for r in runs]


def test_mode0_instructions_per_pipe(compiled):
    # the small-K bn = 128 run, per output: 5 FP32 (exact int -> float, x wscale, x scale_x, + bias, +-0.5), one conversion
    # (F2I), 1/2 LDS (its constants are reread per tile at this width), at most 1/8 store (one may fall past the stretch), and on
    # the ALU pipe one LOP3 (the +-0.5), 1/2 I2IP and one VIMNMX.S16x2 (the clamp on s16 pairs), 1/4 PRMT (the bytes), 1/4 AND
    # (the pad mask) plus the rows' store predicates.  The parent took 6.1 ALU instructions per output here.
    _, sass = compiled
    small = [r for r in mode0_runs(sass, 128) if not any(o.startswith("I2FP") for o in r)]
    assert len(small) == 1
    split = per_pipe(small[0])
    assert split["fp32"] == 5 and split["conversion"] == 1 and split["lds"] == 0.5 and split["store"] <= 1 / 8, split
    assert split["alu"] < 3.5, split
    # the widths up to kConstRegsMaxBN hold their constants in registers: no LDS in their column runs
    for width in range(16, const_regs_max_bn() + 1, 16):
        runs = mode0_runs(sass, width)
        assert runs and not any(o.startswith("LDS") for r in runs for o in r), (width, [per_pipe(r) for r in runs])


def test_small_k_runs_clamp_on_integers(compiled):
    # every small-K run without the border correction clamps the rounded integers (VIMNMX.S16x2), not the floats (FMNMX)
    _, sass = compiled
    runs = [r for r in column_runs(sass) if not any(o.startswith(("LDG", "I2FP")) for o in r)]
    assert len(runs) == 8, len(runs)               # one per width (16 ... 128); layer modes 0 and 1 share it
    assert not any(o.startswith("FMNMX") for r in runs for o in r)
    assert all(any(o.startswith("VIMNMX") for o in r) for r in runs)
