"""Shallow 1x1 layers on the conv-group kernel (conv_group_wgmma.cu, -m gpu): K blocks sized to the layer's K (32 bytes with
32B swizzle and one k-step for Cp <= 32, 64 bytes for Cp <= 64, 128 otherwise) and contiguous multi-tile items read from the
schedule row in shared memory.  Every case reads the plan (mnnb200_conv_int8_group_plan) and the schedule the library deals
for it (mnnb200_conv_group_schedule) and asserts the K block, the K block count and the item lengths it was written for.
Outputs are poisoned first and must equal the C oracle and the mma.sync kernel (variant 1) bit for bit, NHWC16 channel
padding zero."""
import numpy as np
import pytest

from tests.test_conv_group_schedule import schedule
from tests.test_gpu_conv_group import Layer, case, ragged_m
from tests.test_gpu_conv_group_overlap import check_all, sm_count

pytestmark = pytest.mark.gpu


def gemm_layer(backend, rng, ic, oc, tiles, z_in, short=37, relu=0):
    """a 1x1 layer of `tiles` M tiles, the last one `short` rows short of 128"""
    return Layer(backend, case(rng, ic, oc, (1, 1), 1, (1, tiles * 128 - short), relu=relu, z_in=z_in))


def rows_of(layers, sm):
    """the CTA rows the library deals for the layers: lists of (layer, n chunk, first M tile, tiles)"""
    plans = [L.plan() for L in layers]
    return schedule([p["m_tiles"] for p in plans], [p["n_chunks"] for p in plans], sm)


def k_block(cp):
    return 32 if cp <= 32 else (64 if cp <= 64 else 128)


@pytest.mark.parametrize("ic", [13, 29, 40, 64, 75])       # Cp 16, 32, 48, 64, 80
def test_shallow_k_block_by_width(backend, ic):
    # one group per K, a layer per tile width (one-set and two-set widths), each with one or two contiguous tiles per CTA
    sm = sm_count()
    cp = (ic + 15) // 16 * 16
    rng = np.random.default_rng(300 + ic)
    widths = [(13, 16), (45, 48), (64, 64), (90, 96), (128, 128)]
    layers = [gemm_layer(backend, rng, ic, oc, sm + 3 + i, z_in=(-1) ** i * (2 + i), relu=i & 1) for i, (oc, _) in enumerate(widths)]
    for L, (_, bn) in zip(layers, widths):
        p = L.plan()
        assert (p["mode"], p["cb"], p["num_kb"], p["bn"], p["n_chunks"], p["K"]) == (0, k_block(cp), 1, bn, 1, cp), p
        assert ragged_m(L, p) and L.c["z_in"] != 0
    lens = {it[3] for row in rows_of(layers, sm) for it in row}
    assert lens == {1, 2}, lens
    check_all(backend, layers)


@pytest.mark.parametrize("ic,oc", [(16, 16), (32, 61), (20, 96)])
def test_shallow_item_lengths(backend, ic, oc):
    # items of 1, 2, 3, 4 tiles and a range longer than the item's count field holds (65 or 66 tiles: a 64-tile item + the rest)
    sm = sm_count()
    rng = np.random.default_rng(ic * 100 + oc)
    for tiles in (sm + 1, 3 * sm + 5) + ((65 * sm + 3,) if oc == 16 else ()):
        L = gemm_layer(backend, rng, ic, oc, tiles, z_in=-4)
        p = L.plan()
        assert (p["mode"], p["cb"], p["num_kb"], p["m_tiles"]) == (0, 32, 1, tiles) and ragged_m(L, p) and tiles % sm, p
        rows = rows_of([L], sm)
        per_cta = {sum(it[3] for it in row) for row in rows}
        assert per_cta == {tiles // sm, tiles // sm + 1}, per_cta
        if tiles > 64 * sm:
            assert all(len(row) == 2 and row[0][3] == 64 for row in rows)
        else:
            assert all(len(row) == 1 for row in rows)
        check_all(backend, [L])


def test_shallow_mixed_k_blocks_in_one_ring(backend):
    # 32-, 64- and 128-byte K blocks and implicit-GEMM layers (64-byte and 16-byte chunks) back to back in every CTA's row: the
    # stage ring carries stages of different fill and swizzle one after another; a two-chunk layer dealt as single tiles and
    # a layer with fewer tiles than CTAs, whose CTAs change n chunk between items, between range-dealt ones
    sm = sm_count()
    rng = np.random.default_rng(17)
    n_chunks = next(n for n in (3, 5, 7) if sm % n)
    layers = [gemm_layer(backend, rng, 16, 96, 3 * sm + 1, z_in=3, relu=1),                # cb 32, one-set width, 3 / 4 tiles
              gemm_layer(backend, rng, 96, 24, sm + 9, z_in=-2),                           # cb 128
              gemm_layer(backend, rng, 24, 144, sm + 2, z_in=5),                           # cb 32, two chunks of 80: single tiles
              Layer(backend, case(rng, 64, 40, (3, 3), 12, (30, 30), pad=(1, 1), relu=1, z_in=3)),   # mode 1, cb 64
              gemm_layer(backend, rng, 48, 30, 2 * sm + 7, z_in=-3),                       # cb 64, 2 / 3 tiles
              gemm_layer(backend, rng, 32, n_chunks * 112 - 5, sm // 2, z_in=1),           # cb 32, fewer tiles than CTAs
              Layer(backend, case(rng, 24, 45, (3, 3), 8, (20, 20), pad=(1, 1), z_in=-2)),           # mode 1, cb 16
              gemm_layer(backend, rng, 200, 16, sm + 1, z_in=4),                           # cb 128, 2 K blocks
              gemm_layer(backend, rng, 16, 13, 2 * sm - 1, z_in=-5)]                       # cb 32, 1 / 2 tiles
    plans = [L.plan() for L in layers]
    assert [(p["mode"], p["cb"], p["num_kb"]) for p in plans if p["mode"] == 0] == \
        [(0, 32, 1), (0, 128, 1), (0, 32, 1), (0, 64, 1), (0, 32, 1), (0, 128, 2), (0, 32, 1)], plans
    assert [(plans[i]["mode"], plans[i]["cb"]) for i in (3, 6)] == [(1, 64), (1, 16)], plans
    assert (plans[2]["bn"], plans[2]["n_chunks"]) == (80, 2) and plans[5]["n_chunks"] == n_chunks
    rows = rows_of(layers, sm)
    assert len(rows) == sm
    for l, want in ((0, {3, 4}), (1, {1, 2}), (4, {2, 3}), (7, {1, 2}), (8, {1, 2})):
        assert {it[3] for row in rows for it in row if it[0] == l} == want, l
    assert {it[3] for row in rows for it in row if it[0] in (2, 5)} == {1}
    assert any(len({it[1] for it in row if it[0] == 5}) >= 2 for row in rows), "no CTA changes n chunk inside a layer"
    fills = [[plans[it[0]]["cb"] for it in row] for row in rows]
    assert all(len(set(f)) >= 3 for f in fills), "every CTA's ring carries 32-, 64- and 128-byte blocks"
    check_all(backend, layers)


def test_shallow_fewer_items_than_sms(backend):
    # 3 + 2 x 2 = 7 single-tile items of 32-byte K blocks on a grid of 7
    sm = sm_count()
    rng = np.random.default_rng(19)
    layers = [gemm_layer(backend, rng, 16, 16, 3, z_in=2), gemm_layer(backend, rng, 29, 200, 2, z_in=-1)]
    assert [(p["cb"], p["bn"], p["n_chunks"]) for p in (L.plan() for L in layers)] == [(32, 16, 1), (32, 112, 2)]
    rows = rows_of(layers, sm)
    assert len(rows) == 7 < sm and all(len(row) == 1 and row[0][3] == 1 for row in rows)
    check_all(backend, layers)
