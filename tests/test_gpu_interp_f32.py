"""fp32 Interp through the C ABI (-m gpu), against the numpy restatement of the reference CPU (oracle/interp_oracle.py), bit for
bit.  Every recorded golden case, every resize type on both store paths (16-byte stores into an aligned y, scalar stores into a y
4 bytes past 16-byte alignment or with ow % 4 != 0; x between NaN guard bands, y NaN-filled, the path read back through
mnnb200_interp_f32_plan), more than 65,535 planes and rows, one execution resized across shapes against fresh ones, and every
refusal of resize keeping the previous plan."""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import interp_oracle as I
from tests.golden import make_interp_golden as G
from tests.test_gpu_conv_f32 import GUARD, guarded, ptr, sm_count

pytestmark = pytest.mark.gpu
NOT_SUPPORT, NO_EXECUTION = 2, 4
PLAN_FIELDS = ("taps", "vec", "grid", "threads", "row_groups", "x_table", "y_table")
THREADS = 256


def ilib():
    from mnn_b200 import _capi
    return _capi.interp_lib()


def last_error():
    from mnn_b200 import _capi
    return _capi.lib().mnnb200_last_error()


def create(backend, resize_type, transform):
    ws, hs, wo, ho = (float(v) for v in transform)
    h = C.c_void_p()
    assert ilib().mnnb200_interp_f32_create(backend.runtime._h, resize_type, ws, hs, wo, ho, C.byref(h)) == 0, last_error()
    return h


def destroy(h):
    from mnn_b200 import _capi
    _capi.lib().mnnb200_exec_destroy(h)


def plan(h):
    f = (C.c_int * len(PLAN_FIELDS))()
    assert ilib().mnnb200_interp_f32_plan(h, f, len(PLAN_FIELDS)) == 0, last_error()
    return dict(zip(PLAN_FIELDS, f))


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def run(backend, h, x, out_hw, aligned_y=True):
    """execute a resized execution on x (between NaN guard bands, 4 bytes past 16-byte alignment); y aligned (a fresh tensor) or
    guarded like x.  Returns y on the host after checking every guard"""
    import torch
    n, c = x.shape[:2]
    xb, xv = guarded(x.shape, x)
    if aligned_y:
        yb = torch.full((n * c * out_hw[0] * out_hw[1],), float("nan"), dtype=torch.float32, device="cuda")
        yv = yb.view(n, c, *out_hw)
    else:
        yb, yv = guarded((n, c) + tuple(out_hw))
    assert ilib().mnnb200_interp_f32_execute(h, ptr(xv), ptr(yv)) == 0, last_error()
    torch.cuda.synchronize()
    assert torch.isnan(xb[:GUARD]).all() and torch.isnan(xb[-GUARD:]).all()
    if not aligned_y:
        assert torch.isnan(yb[:GUARD]).all() and torch.isnan(yb[-GUARD:]).all(), "a write outside y"
    return yv.cpu().numpy()


def resize(h, n, c, in_hw, out_hw):
    return ilib().mnnb200_interp_f32_resize(h, n * c, in_hw[0], in_hw[1], out_hw[0], out_hw[1])


def expected_plan(resize_type, planes, out_hw, vec):
    taps = {1: 1, 2: 2, 3: 4, 4: 1}[resize_type]
    row_groups = out_hw[1] // 4 if vec else out_hw[1]
    grid = min(16 * sm_count(), math.ceil(planes * out_hw[0] * row_groups / THREADS))
    return dict(taps=taps, vec=int(vec), grid=grid, threads=THREADS, row_groups=row_groups, x_table=out_hw[1] * taps,
                y_table=out_hw[0] * taps)


def check_case(backend, resize_type, transform, x, out_hw, aligned_y=True):
    h = create(backend, resize_type, transform)
    try:
        n, c = x.shape[:2]
        assert resize(h, n, c, x.shape[2:], out_hw) == 0, last_error()
        y = run(backend, h, x, out_hw, aligned_y)
        ref = I.interp(x, resize_type, *transform, out_hw)
        assert np.array_equal(bits(y), bits(ref)), f"{int((bits(y) != bits(ref)).sum())} of {y.size} outputs differ"
        p = plan(h)
        assert p == expected_plan(resize_type, n * c, out_hw, aligned_y and out_hw[1] % 4 == 0), p
        return y
    finally:
        destroy(h)


@pytest.mark.parametrize("name", list(G.CASES))
def test_interp_f32_golden_bit_exact(backend, name):
    """every recorded case (every resize type x coordinate transform): the kernel equals the restatement and the recorded CPU"""
    c = G.CASES[name]
    y = check_case(backend, c["resize_type"], G.case_transform(name), G.case_inputs(name), G.case_out_hw(name))
    shape, sha = G.load()[name]
    assert y.shape == shape and G.digest(y) == sha


SHAPES = [(2, 5, (7, 9), (14, 36)), (1, 6, (9, 10), (17, 24)), (3, 4, (16, 16), (64, 64)), (1, 8, (32, 24), (16, 12)),
          (2, 3, (1, 1), (16, 16)), (1, 5, (9, 7), (3, 4))]


@pytest.mark.parametrize("resize_type", [1, 2, 3, 4])
@pytest.mark.parametrize("ctm", ["AlignCorners", "HalfPixels", "Asymmetric", "TensorflowHalfPixels"])
def test_interp_f32_vector_and_scalar_paths(backend, resize_type, ctm):
    """ow % 4 == 0: 16-byte stores into an aligned y, scalar stores into a y 4 bytes past alignment, the same bits; ow % 4 != 0
    (the second output width) takes the scalar path into an aligned y"""
    rng = np.random.default_rng(resize_type * 10 + len(ctm))
    for n, c, ihw, ohw in SHAPES:
        x = rng.standard_normal((n, c) + ihw).astype(np.float32)
        t = I.transform(resize_type, ctm, 0, 0, ihw, ohw)
        assert np.array_equal(bits(check_case(backend, resize_type, t, x, ohw, True)),
                              bits(check_case(backend, resize_type, t, x, ohw, False)))
        ohw2 = (ohw[0], ohw[1] + 1)
        check_case(backend, resize_type, I.transform(resize_type, ctm, 0, 0, ihw, ohw2), x, ohw2, True)


@pytest.mark.parametrize("resize_type", [1, 2, 3, 4])
def test_interp_f32_many_planes_and_rows(backend, resize_type):
    """70,001 planes (a plane per 3 x 8 output block), and one plane of 70,001 output rows: the grid-stride loop covers both"""
    rng = np.random.default_rng(7 + resize_type)
    x = rng.standard_normal((70001, 1, 2, 3)).astype(np.float32)
    check_case(backend, resize_type, I.transform(resize_type, "HalfPixels", 0, 0, (2, 3), (3, 8)), x, (3, 8))
    x = rng.standard_normal((1, 1, 1000, 5)).astype(np.float32)
    check_case(backend, resize_type, I.transform(resize_type, "AlignCorners", 0, 0, (1000, 5), (70001, 7)), x, (70001, 7))


def test_interp_f32_resized_across_shapes_plans_like_fresh(backend):
    """one execution resized through several shapes: each plan and output equals that of a fresh execution"""
    rng = np.random.default_rng(3)
    t = (0.5, 0.25, -0.25, 0.125)
    h = create(backend, 2, t)
    try:
        for n, c, ihw, ohw in SHAPES + SHAPES[:2]:
            x = rng.standard_normal((n, c) + ihw).astype(np.float32)
            assert resize(h, n, c, ihw, ohw) == 0
            y = run(backend, h, x, ohw)
            f = create(backend, 2, t)
            try:
                assert resize(f, n, c, ihw, ohw) == 0
                assert np.array_equal(bits(run(backend, f, x, ohw)), bits(y))
                assert plan(h) == plan(f)
            finally:
                destroy(f)
    finally:
        destroy(h)


def test_interp_f32_refusals_keep_the_previous_plan(backend):
    """NOT_SUPPORT for an empty tensor and an index past 31 bits, with the previous plan still running; NOT_SUPPORT for resize
    types outside 1-4 and non-finite transforms, whose executions then never run"""
    rng = np.random.default_rng(5)
    x = rng.standard_normal((2, 3, 9, 10)).astype(np.float32)
    t = I.transform(3, "PytorchHalfPixels", 0, 0, (9, 10), (20, 24))
    h = create(backend, 3, t)
    try:
        assert resize(h, 2, 3, (9, 10), (20, 24)) == 0
        before = plan(h)
        run(backend, h, x, (20, 24))
        before = plan(h)
        for args in ((0, 1, (9, 10), (20, 24)), (2, 3, (0, 10), (20, 24)), (2, 3, (9, 10), (20, 0)), (1 << 12, 1, (1 << 10, 1 << 10),
                     (2, 2)), (1, 1, (2, 2), (1 << 16, 1 << 15))):
            assert resize(h, *args) == NOT_SUPPORT, args
            assert plan(h) == before
            y = run(backend, h, x, (20, 24))
            assert np.array_equal(bits(y), bits(I.interp(x, 3, *t, (20, 24))))
    finally:
        destroy(h)
    for resize_type, tr in ((0, t), (5, t), (2, (float("nan"), 1.0, 0.0, 0.0)), (1, (1.0, float("inf"), 0.0, 0.0)),
                            (4, (1.0, 1.0, float("-inf"), 0.0))):
        h = create(backend, resize_type, tr)
        try:
            assert resize(h, 2, 3, (9, 10), (20, 24)) == NOT_SUPPORT, resize_type
            xb, xv = guarded(x.shape, x)
            yb, yv = guarded((2, 3, 20, 24))
            assert ilib().mnnb200_interp_f32_execute(h, ptr(xv), ptr(yv)) == NO_EXECUTION
        finally:
            destroy(h)
