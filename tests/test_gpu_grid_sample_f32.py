"""fp32 GridSample through the C ABI (-m gpu), against the numpy restatement of the reference CPU (oracle/grid_sample_oracle.py),
bit for bit (a NaN only by its position: its sign and payload are the hardware's).  Every recorded golden case; every kernel instantiation on both sides of the channel-group choice and on both grid-read
paths (x and grid 4 bytes off 16-byte alignment between NaN guard bands, y NaN-filled; the plan read back through
mnnb200_grid_sample_f32_plan); the special grid values, a +1e10 coordinate under border padding sampling column 0 as the CPU's
conversion makes it; one execution resized across 4-D and 5-D shapes against fresh ones; every refusal of resize keeping the
previous plan; and a grid of more than 65,535 rows of pixels."""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import grid_sample_oracle as S
from tests.golden import make_grid_sample_golden as G
from tests.test_gpu_conv_f32 import GUARD, guarded, ptr, sm_count

pytestmark = pytest.mark.gpu
NOT_SUPPORT, NO_EXECUTION = 2, 4
PLAN_FIELDS = ("rank", "taps", "cgroups", "cper", "grid", "threads", "vec")
THREADS, FILL = 256, 2048
MODE = {"bilinear": 0, "nearest": 1}
PAD = {"zeros": 0, "border": 1, "reflection": 2}


def glib():
    from mnn_b200 import _capi
    return _capi.grid_sample_lib()


def last_error():
    from mnn_b200 import _capi
    return _capi.lib().mnnb200_last_error()


def create(backend, mode, padding, align):
    h = C.c_void_p()
    assert glib().mnnb200_grid_sample_f32_create(backend.runtime._h, MODE[mode], PAD[padding], int(align), C.byref(h)) == 0, \
        last_error()
    return h


def destroy(h):
    from mnn_b200 import _capi
    _capi.lib().mnnb200_exec_destroy(h)


def plan(h):
    f = (C.c_int * len(PLAN_FIELDS))()
    assert glib().mnnb200_grid_sample_f32_plan(h, f, len(PLAN_FIELDS)) == 0, last_error()
    return dict(zip(PLAN_FIELDS, f))


def bits(a):
    """the fp32 bits of a, every NaN as one pattern: a NaN's sign and payload are the hardware's (x86 gives 0xffc00000 where CUDA
    gives 0x7fffffff), its position is the arithmetic's"""
    a = np.ascontiguousarray(a, np.float32).copy()
    a[np.isnan(a)] = np.float32("nan")
    return a.view(np.uint32)


def golden_digest(y, ref):
    """the digest of y with its NaNs carrying the CPU's bits (ref: the restatement, whose NaNs are x86's), where both are NaN"""
    return G.digest(np.where(np.isnan(y) & np.isnan(ref), ref, y).astype(np.float32))


def resize(h, x_shape, g_shape):
    rank = len(x_shape)
    ind = (C.c_int * (rank - 2))(*x_shape[2:])
    outd = (C.c_int * (rank - 2))(*g_shape[1:-1])
    return glib().mnnb200_grid_sample_f32_resize(h, rank, x_shape[0], x_shape[1], ind, outd)


def run(h, x, g, aligned_grid=False):
    """execute a resized execution: x between NaN guard bands (4 bytes past 16-byte alignment), the grid guarded like x or in a
    fresh (aligned) tensor, y guarded and NaN-filled.  Returns y on the host after checking every guard"""
    import torch
    out_shape = x.shape[:2] + g.shape[1:-1]
    xb, xv = guarded(x.shape, x)
    if aligned_grid:
        gb = gv = torch.from_numpy(np.ascontiguousarray(g, np.float32)).cuda()
    else:
        gb, gv = guarded(g.shape, g)
    yb, yv = guarded(out_shape)
    assert glib().mnnb200_grid_sample_f32_execute(h, ptr(xv), ptr(gv), ptr(yv)) == 0, last_error()
    torch.cuda.synchronize()
    bufs = [(xb, xv, "x"), (yb, yv, "y")] + ([] if aligned_grid else [(gb, gv, "grid")])
    for buf, t, what in bufs:
        band = torch.cat([buf[:GUARD], buf[GUARD + t.numel():]])
        assert bool(torch.isnan(band).all()), f"a write outside {what}"
    return yv.cpu().numpy()


def expected_groups(n, c, pixels):
    groups = min(c, max(1, math.ceil(FILL * sm_count() / (n * pixels))))
    cper = math.ceil(c / groups)
    return math.ceil(c / cper), cper


def sample(backend, x, g, mode, padding, align, aligned_grid=False):
    h = create(backend, mode, padding, align)
    try:
        assert resize(h, x.shape, g.shape) == 0, last_error()
        y = run(h, x, g, aligned_grid)
        return y, plan(h)
    finally:
        destroy(h)


@pytest.mark.parametrize("name", list(G.CASES))
def test_golden_case(backend, name):
    c = G.CASES[name]
    x, g = G.case_inputs(name)
    y, p = sample(backend, x, g, c["mode"], c["padding"], c["align"])
    shape, sha = G.load()[name]
    ref = G.case_oracle(name)
    assert np.array_equal(bits(y), bits(ref))
    assert y.shape == shape and golden_digest(y, ref) == sha
    assert p["rank"] == c["rank"] and p["vec"] == 0


# (n, c, in spatial, out spatial): a few pixels and many channels (grouped), and many pixels and few channels (one group)
FEW_PIXELS = {4: (2, 96, (9, 11), (6, 7)), 5: (2, 40, (5, 6, 7), (2, 3, 4))}
MANY_PIXELS = {4: (2, 3, (40, 50), (400, 420)), 5: (1, 3, (9, 9, 9), (4, 300, 330))}


def _inputs(rng, n, c, ind, outd):
    x = (rng.standard_normal((n, c) + ind) * 2).astype(np.float32)
    g = rng.uniform(-1.15, 1.15, (n,) + outd + (len(ind),)).astype(np.float32)
    g.reshape(-1)[:len(G.SPECIALS)] = np.array(G.SPECIALS, np.float32)
    return x, g


@pytest.mark.parametrize("rank", [4, 5])
@pytest.mark.parametrize("mode", ["bilinear", "nearest"])
@pytest.mark.parametrize("padding", ["zeros", "border"])
def test_every_instantiation_both_channel_groupings(backend, rank, mode, padding):
    """each kernel <rank, mode, padding> on a shape the resize splits into channel groups and on one it runs as one group (both
    alignCorners conventions, both grid-read paths for rank 4), every output equal to the restatement"""
    rng = np.random.default_rng(rank * 100 + len(mode) * 10 + len(padding))
    taps = 1 if mode == "nearest" else (4 if rank == 4 else 8)
    for (n, c, ind, outd), grouped, align in ((FEW_PIXELS[rank], True, False), (MANY_PIXELS[rank], False, True)):
        x, g = _inputs(rng, n, c, ind, outd)
        want = S.grid_sample(x, g, mode, padding, align)
        pixels = int(np.prod(outd))
        groups, cper = expected_groups(n, c, pixels)
        for aligned_grid in ((False, True) if rank == 4 else (False,)):
            y, p = sample(backend, x, g, mode, padding, align, aligned_grid)
            assert np.array_equal(bits(y), bits(want)), (rank, mode, padding, grouped, aligned_grid)
            assert (p["cgroups"], p["cper"]) == (groups, cper)
            assert (p["cgroups"] > 1) == grouped, p
            assert (p["rank"], p["taps"], p["threads"]) == (rank, taps, THREADS)
            assert p["grid"] == min(16 * sm_count(), math.ceil(n * groups * pixels / THREADS))
            assert p["vec"] == (1 if aligned_grid else 0)


def test_special_grid_values(backend):
    """+-1e10, +-Inf and NaN convert to INT_MIN as on x86: under border padding a +1e10 coordinate samples column 0 (not the
    last column a saturating conversion would give), NaN propagates through the weights, and the restatement holds for all"""
    rng = np.random.default_rng(7)
    x = (rng.standard_normal((1, 4, 5, 6)) * 2).astype(np.float32)
    g = np.zeros((1, 1, 8, 2), np.float32)
    g[0, 0, :, 0] = [1e10, -1e10, np.inf, -np.inf, np.nan, 1.0, -1.0, -0.0]
    for mode in ("nearest", "bilinear"):
        for padding in ("zeros", "border"):
            y, _ = sample(backend, x, g, mode, padding, False)
            assert np.array_equal(bits(y), bits(S.grid_sample(x, g, mode, padding, False))), (mode, padding)
    y, _ = sample(backend, x, g, "nearest", "border", False)
    # grid y = 0 -> row (ih - 1) / 2 = 2.0 (+ 0.5 -> floor 2); x = +1e10 -> INT_MIN -> clamped to column 0
    assert np.array_equal(y[0, :, 0, 0], x[0, :, 2, 0])
    assert np.array_equal(y[0, :, 0, 1], x[0, :, 2, 0])
    y, _ = sample(backend, x, g, "bilinear", "zeros", False)
    assert np.isnan(y[0, :, 0, 4]).all()


def test_resize_across_ranks_matches_fresh(backend):
    """one execution resized 4-D -> 5-D -> 4-D, each run equal to a fresh execution's"""
    rng = np.random.default_rng(11)
    shapes = [(2, 7, (6, 8), (9, 5)), (1, 5, (4, 5, 6), (3, 2, 7)), (3, 33, (12, 10), (4, 4))]
    h = create(backend, "bilinear", "zeros", True)
    try:
        for n, c, ind, outd in shapes:
            x, g = _inputs(rng, n, c, ind, outd)
            assert resize(h, x.shape, g.shape) == 0, last_error()
            y = run(h, x, g)
            fresh, p_fresh = sample(backend, x, g, "bilinear", "zeros", True)
            assert np.array_equal(bits(y), bits(fresh))
            assert plan(h) == p_fresh
            assert np.array_equal(bits(y), bits(S.grid_sample(x, g, "bilinear", "zeros", True)))
    finally:
        destroy(h)


def test_resize_refusals_keep_the_plan(backend):
    rng = np.random.default_rng(13)
    x, g = _inputs(rng, 2, 5, (6, 7), (4, 3))
    h = create(backend, "nearest", "border", False)
    try:
        assert glib().mnnb200_grid_sample_f32_plan(h, (C.c_int * 7)(), 7) == NO_EXECUTION
        assert resize(h, x.shape, g.shape) == 0, last_error()
        before = plan(h)
        big = 1 << 16
        bad = [
            (3, 2, 5, (6,), (4,)),                           # rank 3
            (6, 2, 5, (2, 2, 2, 2), (2, 2, 2, 2)),           # rank 6
            (4, 0, 5, (6, 7), (4, 3)),                       # empty batch
            (4, 2, 0, (6, 7), (4, 3)),                       # empty channels
            (4, 2, 5, (0, 7), (4, 3)),                       # empty input
            (4, 2, 5, (6, 7), (4, 0)),                       # empty output
            (4, 2, 5, (big, big), (4, 3)),                   # x past 31 bits
            (4, 2, 5, (6, 7), (big, big)),                   # grid and y past 31 bits
            (5, 1, 1, (6, 7, 8), (1024, 1024, 1025)),        # the grid past 31 bits, 5-D
        ]
        for rank, n, c, ind, outd in bad:
            st = glib().mnnb200_grid_sample_f32_resize(h, rank, n, c, (C.c_int * len(ind))(*ind), (C.c_int * len(outd))(*outd))
            assert st == NOT_SUPPORT, (rank, n, c, ind, outd)
            assert plan(h) == before
        y = run(h, x, g)
        assert np.array_equal(bits(y), bits(S.grid_sample(x, g, "nearest", "border", False)))
    finally:
        destroy(h)


def test_create_refuses_unknown_mode_and_padding(backend):
    h = C.c_void_p()
    assert glib().mnnb200_grid_sample_f32_create(backend.runtime._h, 2, 0, 0, C.byref(h)) == NOT_SUPPORT
    assert glib().mnnb200_grid_sample_f32_create(backend.runtime._h, 0, 3, 0, C.byref(h)) == NOT_SUPPORT


def test_more_than_65535_rows_of_pixels(backend):
    """an output of 70,000 rows: the flat grid-stride launch has no per-dimension grid limit"""
    rng = np.random.default_rng(17)
    x, g = _inputs(rng, 1, 2, (5, 6), (70000, 3))
    for mode in ("bilinear", "nearest"):
        y, _ = sample(backend, x, g, mode, "zeros", False, aligned_grid=True)
        assert np.array_equal(bits(y), bits(S.grid_sample(x, g, mode, "zeros", False))), mode
