"""The conv-group kernel's run walk and next-tile overlap (conv_group_wgmma.cu, -m gpu).  A consumer warpgroup walks runs of
consecutive same-(layer, n chunk) items of its schedule row; for tile widths up to kOverlapMaxBN (64) it issues the next
tile's first K block into a second accumulator set before the current tile's epilogue when that tile's stage has already
landed.  The cases give runs of 1, 2 and odd / even many tiles per CTA (M derived from the device's SM count), switches
between two-set and one-set widths inside a CTA's row, K of several blocks, part-empty last M tiles, a group with fewer
items than SMs, CTAs whose n chunk changes between items (widths >= 80: group_bn gives one chunk up to 128 padded channels)
and an implicit-GEMM 3x3 layer with z_in != 0 and border correction.  Outputs are poisoned first and must equal the C oracle
and the mma.sync kernel (variant 1) bit for bit, NHWC16 channel padding zero."""
import numpy as np
import pytest

from tests.test_conv_group_overlap_sass import overlap_max_bn
from tests.test_gpu_conv_group import Layer, case, ragged_m, ragged_n, run_group, schedule

pytestmark = pytest.mark.gpu

OVERLAP_MAX_BN = overlap_max_bn()


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def gemm_layer(backend, rng, ic, oc, tiles, short=37, relu=0):
    """a 1x1 layer of `tiles` M tiles, the last one `short` rows short of 128"""
    return Layer(backend, case(rng, ic, oc, (1, 1), 1, (1, tiles * 128 - short), relu=relu, z_in=int(rng.integers(-5, 6))))


def check_all(backend, layers):
    refs = [L.submit() for L in layers]
    run_group(backend, layers)
    grouped = [L.check(r.result()) for L, r in zip(layers, refs)]
    for L, y in zip(layers, grouped):
        L.ex.set_variant(1)
        L.poison()
        assert L.ex.onExecute([L.xin], [L.yout]) == 0
        backend.onSync()
        assert np.array_equal(L.output(), y), ("variant 1", L.plan())


def run_lengths(layers, sm):
    """for every CTA row, the lengths of its runs of same-(layer, n chunk) items"""
    out = []
    for row in schedule(layers, sm):
        runs, prev = [], None
        for it in row:
            if it == prev:
                runs[-1] += 1
            else:
                runs.append(1)
            prev = it
        out.append(runs)
    return out


@pytest.mark.parametrize("bn", [16, 32, 48, 64])
def test_overlap_run_lengths_one_layer(backend, bn):
    sm = sm_count()
    rng = np.random.default_rng(100 + bn)
    for tiles in (sm + 1, 2 * sm + 1, 3 * sm - 1):      # runs of (2, 1), (3, 2), (3, 2) tiles per CTA
        L = gemm_layer(backend, rng, 48, bn - 3, tiles)
        p = L.plan()
        assert (p["mode"], p["bn"], p["n_chunks"], p["m_tiles"]) == (0, bn, 1, tiles) and ragged_m(L, p), p
        lens = {n for r in run_lengths([L], sm) for n in r}
        assert {tiles // sm, tiles // sm + 1} == lens, lens
        check_all(backend, [L])


def test_overlap_width_switches_and_long_k(backend):
    # two-set widths with 2 and 5 K blocks (K 144, 576) and an implicit-GEMM 3x3 layer, between one-set widths: every CTA's
    # row switches from a two-set run to a one-set run and back
    sm = sm_count()
    rng = np.random.default_rng(7)
    layers = [gemm_layer(backend, rng, 144, 61, sm + 5, relu=1),         # bn 64, 2 K blocks
              gemm_layer(backend, rng, 64, 128, sm + 1),                 # bn 128
              gemm_layer(backend, rng, 576, 30, 2 * sm - 3),             # bn 32, 5 K blocks
              gemm_layer(backend, rng, 32, 140, sm // 2 + 3),            # bn 80, 2 chunks, ragged
              Layer(backend, case(rng, 32, 45, (3, 3), 24, (36, 36), pad=(1, 1), relu=1, z_in=3)),   # bn 48, mode 1
              gemm_layer(backend, rng, 16, 14, sm + 7)]                  # bn 16
    plans = [L.plan() for L in layers]
    assert [p["bn"] for p in plans] == [64, 128, 32, 80, 48, 16], plans
    assert [p["num_kb"] for p in plans][:3] == [2, 1, 5], plans
    assert ragged_n(layers[3], plans[3]) and plans[3]["n_chunks"] == 2
    p3 = plans[4]
    assert p3["mode"] == 1 and p3["m_tiles"] > sm and layers[4].c["z_in"] != 0, p3
    two = {l for l, p in enumerate(plans) if p["bn"] <= OVERLAP_MAX_BN}
    switches = 0
    for row in schedule(layers, sm):
        kinds = [it[0] in two for it in row]
        switches += sum(a != b for a, b in zip(kinds, kinds[1:]))
    assert switches >= 2 * sm, switches
    check_all(backend, layers)


def test_overlap_fewer_items_than_sms(backend):
    # 3 + 2 x 2 = 7 items: grid 7, one item (a run of 1) per CTA, the grid not a multiple of the second layer's n chunks
    sm = sm_count()
    rng = np.random.default_rng(11)
    layers = [gemm_layer(backend, rng, 32, 32, 3), gemm_layer(backend, rng, 32, 200, 2)]
    assert [(p["bn"], p["n_chunks"]) for p in (L.plan() for L in layers)] == [(32, 1), (112, 2)]
    assert len(schedule(layers, sm)) == 7 < sm
    check_all(backend, layers)


def test_overlap_n_chunk_changes_between_items(backend):
    # a layer whose n chunk count does not divide the grid: a CTA's consecutive items of it change n chunk (runs of 1, the
    # constants slot switching at every item), after a two-set run
    sm = sm_count()
    n_chunks = next(n for n in (5, 7, 3) if sm % n)
    rng = np.random.default_rng(13)
    layers = [gemm_layer(backend, rng, 32, 48, sm + 3),
              gemm_layer(backend, rng, 32, n_chunks * 112 - 5, sm // n_chunks + 4)]
    p = layers[1].plan()
    assert (p["bn"], p["n_chunks"]) == (112, n_chunks), p
    changes = 0
    for row in schedule(layers, sm):
        chunks = [it[1] for it in row if it[0] == 1]
        changes += sum(a != b for a, b in zip(chunks, chunks[1:]))
    assert changes > 0
    check_all(backend, layers)
