"""The conv-group kernel's schedule as the library builds it (mnnb200_conv_group_schedule, no GPU needed): every (layer, n
chunk, M tile) is in exactly one item, the CTAs' tile counts differ by at most one per (layer, n chunk), every row keeps the
layers in list order, a one-chunk layer with a tile per CTA is dealt as one contiguous range per CTA and the extra tiles of
such layers do not pile up on the same CTAs."""
import ctypes as C

import pytest

from mnn_b200 import _capi

END = 0xFFFFFFFF


def decode(w):
    """(layer, n chunk, first M tile, tiles)"""
    return w >> 26, (w >> 20) & 63, w & 0x3FFF, ((w >> 14) & 63) + 1


def schedule(m_tiles, n_chunks, sm):
    """the CTA rows, each a list of decoded items"""
    L = len(m_tiles)
    mt, nc = (C.c_int * L)(*m_tiles), (C.c_int * L)(*n_chunks)
    grid, stride = C.c_int(), C.c_int()
    lib = _capi.lib()
    assert lib.mnnb200_conv_group_schedule(mt, nc, L, sm, None, 0, C.byref(grid), C.byref(stride)) == 0
    buf = (C.c_uint32 * (grid.value * stride.value))()
    assert lib.mnnb200_conv_group_schedule(mt, nc, L, sm, buf, len(buf), C.byref(grid), C.byref(stride)) == 0
    rows = []
    for c in range(grid.value):
        row = list(buf[c * stride.value:(c + 1) * stride.value])
        n = row.index(END)
        assert n <= stride.value - 2 and all(w == END for w in row[n:]), "a row ends with at least two end markers"
        rows.append([decode(w) for w in row[:n]])
    return rows


MIXES = [
    ([3136, 3136, 784, 784, 784, 196, 49, 13], [1, 1, 1, 2, 1, 2, 3, 8], 132),     # the shape of MobileNet-v2 at batch 32
    ([133, 265, 395, 132, 131, 700], [1, 1, 1, 1, 1, 1], 132),                     # 1, 2, 3 tiles per CTA, ragged
    ([132 * 64 + 5, 9000, 16383], [1, 2, 1], 132),                                 # ranges longer than one item holds
    ([3, 2], [1, 2], 132),                                                         # fewer items than CTAs
    ([500, 77, 1000], [1, 1, 1], 7),
]


@pytest.mark.parametrize("m_tiles,n_chunks,sm", MIXES)
def test_every_tile_once_and_balanced(m_tiles, n_chunks, sm):
    rows = schedule(m_tiles, n_chunks, sm)
    assert len(rows) == min(sm, sum(t * n for t, n in zip(m_tiles, n_chunks)))
    seen = {}
    for c, row in enumerate(rows):
        assert [it[0] for it in row] == sorted(it[0] for it in row), "layers in list order in every row"
        for l, nc, mt, cnt in row:
            for t in range(mt, mt + cnt):
                assert (l, nc, t) not in seen, (l, nc, t)
                seen[(l, nc, t)] = c
    assert len(seen) == sum(t * n for t, n in zip(m_tiles, n_chunks))
    assert all(t < m_tiles[l] and nc < n_chunks[l] for l, nc, t in seen)
    for l in range(len(m_tiles)):
        per_cta = [sum(cnt for ll, _, _, cnt in row if ll == l) for row in rows]
        assert max(per_cta) - min(per_cta) <= 1, (l, min(per_cta), max(per_cta))
        if n_chunks[l] == 1 and m_tiles[l] >= len(rows):
            # one contiguous range per CTA, in as few items as the 6-bit count field allows
            for row in rows:
                its = [it for it in row if it[0] == l]
                assert all(a[2] + a[3] == b[2] for a, b in zip(its, its[1:])), its
                assert len(its) == -(-sum(it[3] for it in its) // 64), its
        else:
            assert all(cnt == 1 for row in rows for ll, _, _, cnt in row if ll == l)
    total = [sum(cnt for _, _, _, cnt in row) for row in rows]
    assert max(total) - min(total) <= 1, "the extra tiles of successive layers go to different CTAs"


def test_schedule_rejects_bad_arguments():
    lib = _capi.lib()
    g, s = C.c_int(), C.c_int()
    one = (C.c_int * 1)(4)
    assert lib.mnnb200_conv_group_schedule(one, one, 0, 132, None, 0, C.byref(g), C.byref(s)) != 0
    assert lib.mnnb200_conv_group_schedule(one, one, 1, 0, None, 0, C.byref(g), C.byref(s)) != 0
    assert lib.mnnb200_conv_group_schedule((C.c_int * 1)(16384), one, 1, 132, None, 0, C.byref(g), C.byref(s)) != 0
    assert lib.mnnb200_conv_group_schedule(one, (C.c_int * 1)(64), 1, 132, None, 0, C.byref(g), C.byref(s)) != 0
    buf = (C.c_uint32 * 4)()
    assert lib.mnnb200_conv_group_schedule(one, one, 1, 132, buf, 4, C.byref(g), C.byref(s)) != 0      # 16 rows x 3 words needed
