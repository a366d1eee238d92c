"""The conv-group kernel's next-tile overlap (conv_group_wgmma.cu), checked in the SASS ptxas makes for sm_90a without a GPU.  For
tile widths up to kOverlapMaxBN the consumers probe the next tile's stage without blocking (a warpgroup-wide BAR.RED) and, if it
has landed, issue its first K block into a second accumulator set before the current tile's epilogue; wider tiles keep one
set and no probe.  That only pays if ptxas keeps the wgmmas asynchronous (spills: test_conv_group_sass.py)."""
import re

from tests.test_conv_group_sass import CONTROL, SRC, compiled, kernel_instructions, pytestmark  # noqa: F401  (compiled: module fixture)


def overlap_max_bn():
    m = re.search(r"constexpr int kOverlapMaxBN = (\d+);", open(SRC).read())
    assert m, "kOverlapMaxBN not found in " + SRC
    return int(m.group(1))


def column_runs_after_probe(ops):
    """(width, probe, mma) for every epilogue column run: width = 2 x its F2I.TRUNCs; probe = a BAR.RED since the previous
    column run; mma = an IGMMA between that probe and the run"""
    out, probe, mma, i = [], False, False, 0
    while i < len(ops):
        op = ops[i]
        if op.startswith("BAR.RED"):
            probe, mma = True, False
        elif op.startswith("IGMMA"):
            mma = mma or probe
        elif op.startswith("F2I.TRUNC"):
            n = 0
            while i < len(ops) and not ops[i].startswith(CONTROL):
                n += ops[i].startswith("F2I.TRUNC")
                i += 1
            out.append((2 * n, probe, mma))
            probe, mma = False, False
            continue
        i += 1
    return out


def test_no_wgmma_serialization(compiled):
    ptxas, _ = compiled
    assert "wgmma.mma_async instructions are serialized" not in ptxas, ptxas


def test_next_tile_mma_issued_before_epilogue(compiled):
    # every overlapped width has a column run reached from a probe with the next tile's IGMMA in between; no probe leads to a
    # wider tile's column run
    _, sass = compiled
    limit = overlap_max_bn()
    runs = column_runs_after_probe(kernel_instructions(sass))
    probed = [(w, mma) for w, probe, mma in runs if probe]
    assert all(mma for _, mma in probed), probed
    assert {w for w, _ in probed} == set(range(16, limit + 1, 16)), sorted(set(probed))


def test_wide_tiles_keep_one_set(compiled):
    # bn > kOverlapMaxBN: column runs exist for every such width and none follows a probe
    _, sass = compiled
    limit = overlap_max_bn()
    runs = column_runs_after_probe(kernel_instructions(sass))
    wide = [(w, probe) for w, probe, _ in runs if w > limit]
    assert {w for w, _ in wide} >= set(range(limit + 16, 129, 16)), sorted(set(wide))
    assert not any(probe for _, probe in wide), wide
