"""The shallow conv-group kernel (conv_group_shallow_wgmma.cu, -m gpu): 1x1 layers of one K block at tile widths up to
kGroupShallowMaxBN, their 64-row halves dealt to four consumer warpgroups.  Every case reads the kernel the plan chose (the last
field of mnnb200_conv_int8_group_plan: 0 the conv-group kernel, 1 the shallow one).  Outputs are poisoned first and must equal
the C oracle and the mma.sync kernel (variant 1) bit for bit, NHWC16 channel padding zero."""
import ctypes as C

import numpy as np
import pytest

from tests.test_conv_group_shallow_sass import shallow_max_bn
from tests.test_gpu_conv_group import Layer, case, ragged_m
from tests.test_gpu_conv_group_overlap import check_all, sm_count

pytestmark = pytest.mark.gpu


def kernel(L):
    from mnn_b200 import _capi
    f = (C.c_int * 11)()
    assert _capi.lib().mnnb200_conv_int8_group_plan(L.ex._h, f, 11) == 0
    return f[10]


def gemm_layer(backend, rng, ic, oc, rows, z_in, relu=0, z_out=None):
    c = case(rng, ic, oc, (1, 1), 1, (1, rows), relu=relu, z_in=z_in)
    if z_out is not None:
        c["z_out"] = z_out
    return Layer(backend, c)


@pytest.mark.parametrize("ic,cb", [(13, 32), (29, 32), (40, 64), (64, 64), (75, 128), (128, 128)])
def test_every_width_and_k_block(backend, ic, cb):
    # one group per K block, a member per width 16 ... 96 (four of them ragged in N): 4 x #SMs + 3 M tiles, the last one 37
    # rows short, so the 64-row halves do not divide evenly over the warpgroups and the last half is empty
    sm = sm_count()
    rng = np.random.default_rng(500 + ic)
    widths = [(13, 16), (32, 32), (45, 48), (64, 64), (70, 80), (90, 96)]
    assert widths[-1][1] == shallow_max_bn()
    layers = [gemm_layer(backend, rng, ic, oc, (4 * sm + 3) * 128 - 37, z_in=(-1) ** i * (2 + i), relu=i & 1)
              for i, (oc, _) in enumerate(widths)]
    for L, (_, bn) in zip(layers, widths):
        p = L.plan()
        assert (p["mode"], p["cb"], p["num_kb"], p["bn"], p["n_chunks"]) == (0, cb, 1, bn, 1), p
        assert ragged_m(L, p) and kernel(L) == 1
    check_all(backend, layers)


@pytest.mark.parametrize("rows", [50, 64, 128 + 20, 3 * 64 + 5])
def test_few_half_tiles(backend, rows):
    # a single half tile (M <= 64), one whole M tile, and one and a half tiles: warpgroups with no half at all
    rng = np.random.default_rng(rows)
    layers = [gemm_layer(backend, rng, 24, 40, rows, z_in=3), gemm_layer(backend, rng, 96, 24, rows, z_in=-2, relu=1)]
    assert [kernel(L) for L in layers] == [1, 1]
    check_all(backend, layers)


def test_half_counts_over_the_grid(backend):
    # M tiles 1 short of, equal to and 1 past whole rounds of 4 warpgroups x #SMs halves, and contiguous multi-tile items
    sm = sm_count()
    rng = np.random.default_rng(41)
    layers = [gemm_layer(backend, rng, 16, 96, tiles * 128 - 11, z_in=-1 - i)
              for i, tiles in enumerate((2 * sm - 1, 2 * sm, 2 * sm + 1, 5 * sm + 2))]
    assert all(kernel(L) == 1 for L in layers)
    check_all(backend, layers)


def test_n_chunks_change_between_tiles(backend):
    # two chunks of 80 (24 -> 144) and of 96 (32 -> 192), and three chunks of 96 on fewer M tiles than CTAs, whose CTAs change
    # n chunk from item to item: every warpgroup's weight slot alternates between runs
    sm = sm_count()
    rng = np.random.default_rng(43)
    layers = [gemm_layer(backend, rng, 24, 144, (sm + 2) * 128 - 9, z_in=5),
              gemm_layer(backend, rng, 32, 192, (sm // 2) * 128 - 3, z_in=-4, relu=1),
              gemm_layer(backend, rng, 64, 270, (sm // 2 + 1) * 128 - 70, z_in=2)]
    assert [(L.plan()["bn"], L.plan()["n_chunks"], kernel(L)) for L in layers] == [(80, 2, 1), (96, 2, 1), (96, 3, 1)]
    check_all(backend, layers)


def test_clamp_without_zero_clears_pad_channels(backend):
    # ReLU with z_out > 0: the clamp excludes 0, so the pad channels of the last chunk are cleared by the byte masks
    sm = sm_count()
    rng = np.random.default_rng(47)
    layers = [gemm_layer(backend, rng, 40, oc, (sm + 5) * 128 - 21, z_in=-3, relu=1, z_out=zo)
              for oc, zo in ((45, 6), (21, 3), (150, 9))]
    assert all(kernel(L) == 1 and L.oc % 16 for L in layers)
    check_all(backend, layers)


def test_mixed_group_runs_both_kernels(backend):
    # shallow members next to a 128-wide one, a two-K-block one and an implicit-GEMM 3x3: two launches, the conv-group kernel's
    # after the shallow kernel's
    from mnn_b200.backend import ConvGroupExecution
    sm = sm_count()
    rng = np.random.default_rng(53)
    layers = [gemm_layer(backend, rng, 16, 96, (3 * sm + 1) * 128 - 5, z_in=3, relu=1),
              gemm_layer(backend, rng, 64, 128, (sm + 3) * 128 - 17, z_in=-2),
              gemm_layer(backend, rng, 96, 24, (sm + 9) * 128 - 30, z_in=4),
              gemm_layer(backend, rng, 200, 32, (sm + 1) * 128 - 7, z_in=-5),
              Layer(backend, case(rng, 64, 40, (3, 3), 4, (30, 30), pad=(1, 1), relu=1, z_in=3))]
    assert [kernel(L) for L in layers] == [1, 0, 1, 0, 0]
    grp = ConvGroupExecution(backend, [L.ex for L in layers])
    assert grp.launches() == 2
    check_all(backend, layers)
    only_wide = ConvGroupExecution(backend, [layers[1].ex, layers[3].ex])
    assert only_wide.launches() == 1
