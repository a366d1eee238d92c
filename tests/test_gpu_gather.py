"""The gathers, the casts and the broadcast float MatMul through the C ABI (-m gpu).  Every recorded gather and cast golden bit for
bit (and equal to the numpy restatement); both store paths of the slice gather (16-byte: inside % 4 == 0 and aligned tensors;
4-byte: a params or output 4 bytes past 16-byte alignment, or inside % 4 != 0) with NaN guard bands around the output; more than
65,535 slices and slices longer than one tile; one execution resized across shapes; refusals that keep the previous plan; and the
broadcast MatMul goldens within 1e-3 of max|ref|, with create_broadcast equal to create where nothing broadcasts."""
import ctypes as C

import numpy as np
import pytest

from oracle import gather_oracle as G
from tests.golden import make_gather_golden as M
from tests.test_gpu_conv_f32 import GUARD, ptr

pytestmark = pytest.mark.gpu
NOT_SUPPORT = 2
PLAN_FIELDS = ("mode", "path", "grid", "threads", "slices_per_tile", "outside", "n", "inside")
MODES = {"Gather": 0, "GatherV2": 0, "GatherND": 1, "GatherElements": 2}


def glib():
    from mnn_b200 import _capi
    return _capi.gather_lib()


def last_error():
    from mnn_b200 import _capi
    return _capi.lib().mnnb200_last_error()


def destroy(h):
    from mnn_b200 import _capi
    _capi.lib().mnnb200_exec_destroy(h)


def ints(v):
    v = list(v) or [1]
    return (C.c_int * len(v))(*v), len(v)


def create(backend, mode):
    h = C.c_void_p()
    assert glib().mnnb200_gather_create(backend.runtime._h, mode, C.byref(h)) == 0, last_error()
    return h


def resize(h, pshape, ishape, axis):
    pd, pr = ints(pshape)
    idd, ir = ints(ishape)
    return glib().mnnb200_gather_resize(h, pd, pr, idd, ir, int(axis))


def plan(h):
    f = (C.c_int * len(PLAN_FIELDS))()
    assert glib().mnnb200_gather_plan(h, f, len(PLAN_FIELDS)) == 0, last_error()
    return dict(zip(PLAN_FIELDS, f))


def dev(a, offset=0):
    """(buffer, view): a as 4-byte words on the device, `offset` words past a 16-byte aligned start, NaN-guarded"""
    import torch
    a = np.ascontiguousarray(a)
    words = torch.from_numpy(a.view(np.int32).reshape(-1).copy())
    buf = torch.full((a.size + 2 * GUARD + offset,), -1, dtype=torch.int32, device="cuda")
    start = GUARD + offset - (GUARD % 4)                        # GUARD % 4 == 1: start is offset words past alignment
    view = buf[start:start + a.size]
    view.copy_(words)
    assert view.data_ptr() % 16 == 4 * (offset % 4)
    return buf, view, start


def run(h, params, indices, out_shape, out_dtype, p_off=0, y_off=0):
    import torch
    _, pv, _ = dev(params, p_off)
    _, iv, _ = dev(np.asarray(indices, np.int32).reshape(-1) if np.asarray(indices).ndim else np.asarray(indices, np.int32).reshape(1))
    count = int(np.prod(out_shape))
    yb, yv, start = dev(np.full(count, -7, np.int32), y_off)
    assert glib().mnnb200_gather_execute(h, ptr(pv), ptr(iv), ptr(yv)) == 0, last_error()
    torch.cuda.synchronize()
    host = yb.cpu().numpy()
    assert (host[:start] == -1).all() and (host[start + count:] == -1).all(), "a write outside the output"
    return host[start:start + count].view(out_dtype).reshape(out_shape)


def gather_case(backend, name, p_off=0, y_off=0):
    c = M.CASES[name]
    params, idx = M.case_inputs(name)
    axis = c["axis"] or 0
    h = create(backend, MODES[c["kind"]])
    try:
        assert resize(h, params.shape, idx.shape if idx.ndim else (1,), axis) == 0, last_error()
        ref = M.case_oracle(name)
        y = run(h, params, idx, ref.shape, params.dtype, p_off, y_off)
        return y, ref, plan(h)
    finally:
        destroy(h)


@pytest.mark.parametrize("name", [n for n in M.CASES if M.CASES[n]["kind"] != "Cast"])
def test_golden_gathers_bit_exact(backend, name):
    y, ref, pl = gather_case(backend, name)
    shape, sha = M.load()[0][name]
    assert y.shape == shape and M.digest(y) == sha
    assert np.array_equal(y.view(np.uint32), ref.view(np.uint32))
    assert pl["mode"] == MODES[M.CASES[name]["kind"]] and pl["threads"] == 256 and pl["grid"] >= 1


def test_casts_bit_exact(backend):
    import torch
    L = glib()
    rt = backend.runtime._h
    for name, fn, out in (("cast_i32_f32", L.mnnb200_cast_i32_f32, np.float32), ("cast_f32_i32", L.mnnb200_cast_f32_i32, np.int32)):
        x = M.case_inputs(name)[0]
        for off in (0, 1):
            _, xv, _ = dev(x, off)
            yb, yv, start = dev(np.zeros(x.size, np.int32), off)
            assert fn(rt, ptr(xv), ptr(yv), x.size) == 0, last_error()
            torch.cuda.synchronize()
            host = yb.cpu().numpy()
            assert (host[:start] == -1).all() and (host[start + x.size:] == -1).all()
            y = host[start:start + x.size].view(out)
            assert M.digest(y) == M.load()[0][name][1], (name, off)
        assert fn(rt, None, None, 0) == 0
        assert fn(rt, None, None, -1) != 0


@pytest.mark.parametrize("inside", [1, 3, 4, 768, 20000])
def test_gather_store_paths(backend, inside):
    """each slice length on the aligned tensors (16-byte when inside % 4 == 0) and with params / output 4 bytes past alignment
    (4-byte); 20000 is longer than a tile (several chunks per slice)"""
    rng = np.random.default_rng(inside)
    rows = 37
    params = rng.standard_normal((3, rows, inside)).astype(np.float32)
    idx = rng.integers(-2, rows + 2, (5,)).astype(np.int32)
    ref = G.gather(params, idx, 1)
    h = create(backend, 0)
    try:
        assert resize(h, params.shape, idx.shape, 1) == 0, last_error()
        for p_off, y_off in ((0, 0), (1, 0), (0, 1)):
            y = run(h, params, idx, ref.shape, np.float32, p_off, y_off)
            assert np.array_equal(y.view(np.uint32), ref.view(np.uint32)), (p_off, y_off)
            pl = plan(h)
            assert pl["path"] == (1 if inside % 4 == 0 and p_off == 0 and y_off == 0 else 0), pl
            assert (pl["outside"], pl["n"], pl["inside"]) == (3, 5, inside)
    finally:
        destroy(h)


def test_more_than_65535_slices(backend):
    rng = np.random.default_rng(3)
    params = rng.standard_normal((1000, 3)).astype(np.float32)
    idx = rng.integers(-5, 1005, (70000 * 2,)).astype(np.int32)
    ref = G.gather(params, idx, 0)
    nd_idx = rng.integers(0, 1000, (100000, 1)).astype(np.int32)
    for mode, p, i, r, axis in ((0, params, idx, ref, 0), (1, params, nd_idx, G.gather_nd(params, nd_idx), 0)):
        h = create(backend, mode)
        try:
            assert resize(h, p.shape, i.shape, axis) == 0, last_error()
            y = run(h, p, i, r.shape, np.float32)
            assert np.array_equal(y.view(np.uint32), r.view(np.uint32))
            assert plan(h)["n"] == int(np.prod(i.shape[:-1] if mode == 1 else i.shape))
        finally:
            destroy(h)
    # GatherElements over 280,000 elements, more than the capped grid's threads: the grid-stride loop
    big = rng.standard_normal((4, 70000)).astype(np.float32)
    el = rng.integers(-1, 70001, (4, 70000)).astype(np.int32)
    h = create(backend, 2)
    try:
        assert resize(h, big.shape, el.shape, 1) == 0
        y = run(h, big, el, el.shape, np.float32)
        assert np.array_equal(y, G.gather_elements(big, el, 1))
    finally:
        destroy(h)


def test_resize_across_shapes_and_refusals_keep_the_plan(backend):
    rng = np.random.default_rng(11)
    h = create(backend, 0)
    try:
        for shape, ishape, axis in (((6, 8), (4,), 0), ((2, 9, 16), (3, 2), 1), ((5, 4), (7,), -1), ((6, 8), (4,), 0)):
            params = rng.standard_normal(shape).astype(np.float32)
            idx = rng.integers(0, shape[axis], ishape).astype(np.int32)
            assert resize(h, shape, ishape, axis) == 0
            y = run(h, params, idx, G.gather(params, idx, axis).shape, np.float32)
            assert np.array_equal(y, G.gather(params, idx, axis))
        before = plan(h)
        for bad in (((6, 0), (4,), 0), ((6, 8), (0,), 0), ((6, 8), (4,), 2), ((6, 8), (4,), -3), ((1,) * 9, (4,), 0),
                    ((70000, 40000), (4,), 0)):
            assert resize(h, *bad) == NOT_SUPPORT, bad
            assert plan(h) == before, bad
        params = rng.standard_normal((6, 8)).astype(np.float32)
        idx = rng.integers(0, 6, (4,)).astype(np.int32)
        assert np.array_equal(run(h, params, idx, (4, 8), np.float32), G.gather(params, idx, 0))
    finally:
        destroy(h)
    h = create(backend, 1)
    try:
        assert resize(h, (3, 4, 5), (2, 2), 0) == 0
        before = plan(h)
        for bad in (((3, 4, 5), (2, 4), 0), ((3, 4, 5), (2, 2), 2), ((3, 4, 5), (2, 2), -1), ((3, 4, 5), (2, 3), 1)):
            assert resize(h, *bad) == NOT_SUPPORT, bad
            assert plan(h) == before, bad
    finally:
        destroy(h)
    h = create(backend, 2)
    try:
        assert resize(h, (3, 4), (3, 2), 0) == 0
        before = plan(h)
        for bad in (((3, 4), (3, 2, 1), 0), ((3, 4), (3, 5), 0), ((3, 4), (3, 2), 2)):
            assert resize(h, *bad) == NOT_SUPPORT, bad
            assert plan(h) == before, bad
    finally:
        destroy(h)


def _matmul(backend, a, b, ta, tb, broadcast=True):
    """(C, handle created) of one MatMul through mnnb200_matmul_create_broadcast, with ShapeMatMul's dims and 1-D squeeze"""
    import torch
    from mnn_b200 import _capi
    L = _capi.lib()
    na, nb = a.ndim, b.ndim
    ta, tb = na > 1 and ta, nb == 1 or tb
    e = 1 if na == 1 else (a.shape[-1] if ta else a.shape[-2])
    l = a.shape[0] if na == 1 else (a.shape[-2] if ta else a.shape[-1])
    h = 1 if nb == 1 else (b.shape[-2] if tb else b.shape[-1])
    ba, bb = a.shape[:-2], b.shape[:-2]
    nd = max(len(ba), len(bb))
    ad = (1,) * (nd - len(ba)) + tuple(ba)
    bd = (1,) * (nd - len(bb)) + tuple(bb)
    cd = tuple(max(x, y) for x, y in zip(ad, bd))
    hdl = C.c_void_p()
    arr = lambda v: (C.c_int * max(len(v), 1))(*v)   # noqa: E731
    if broadcast:
        st = L.mnnb200_matmul_create_broadcast(backend.runtime._h, nd, arr(cd), arr(ad), arr(bd), e, l, h, int(ta), int(tb),
                                               C.byref(hdl))
    else:
        st = L.mnnb200_matmul_create(backend.runtime._h, int(np.prod(cd)), e, l, h, int(ta), int(tb), 0, C.byref(hdl))
    assert st == 0, last_error()
    try:
        at, bt = torch.from_numpy(np.ascontiguousarray(a)).cuda(), torch.from_numpy(np.ascontiguousarray(b)).cuda()
        c = torch.full(cd + (e, h), float("nan"), dtype=torch.float32, device="cuda")
        assert L.mnnb200_matmul_execute(hdl, ptr(at), ptr(bt), None, ptr(c)) == 0, last_error()
        torch.cuda.synchronize()
        return c.cpu().numpy()
    finally:
        L.mnnb200_exec_destroy(hdl)


@pytest.mark.parametrize("name", list(M.MATMUL_CASES))
def test_broadcast_matmul_goldens(backend, name):
    _, _, _, ta, tb = M.MATMUL_CASES[name]
    a, b = M.case_inputs(name)
    ref = M.load()[1][name]
    y = _matmul(backend, a, b, ta, tb).reshape(ref.shape)
    assert np.abs(y - ref).max() <= 1e-3 * np.abs(ref).max()


def test_broadcast_matmul_attention_shapes_and_no_broadcast_equals_create(backend):
    rng = np.random.default_rng(5)
    a = rng.standard_normal((4, 12, 128, 64)).astype(np.float32)
    b = rng.standard_normal((4, 12, 128, 64)).astype(np.float32)
    y1 = _matmul(backend, a, b, 0, 1)
    y0 = _matmul(backend, a, b, 0, 1, broadcast=False)
    assert np.array_equal(y0.view(np.uint32), y1.view(np.uint32))
    ref = np.matmul(a.astype(np.float64), np.swapaxes(b, -1, -2).astype(np.float64))
    assert np.abs(y1 - ref).max() <= 1e-3 * np.abs(ref).max()
    w = rng.standard_normal((768, 300)).astype(np.float32)
    x = rng.standard_normal((3, 200, 768)).astype(np.float32)
    ref = x.astype(np.float64) @ w
    y = _matmul(backend, x, w, 0, 0)
    assert np.abs(y - ref).max() <= 1e-3 * np.abs(ref).max()


@pytest.mark.parametrize("kind,axis", [("Gather", 1), ("GatherND", 1), ("GatherElements", -1)])
def test_python_mirror_gather(backend, kind, axis):
    """Op(type="Gather" / "GatherND" / "GatherElements") through the Python mirror's creator: shape and values"""
    import torch
    from mnn_b200.backend import Op, Tensor
    rng = np.random.default_rng(13)
    params = rng.standard_normal((3, 6, 5)).astype(np.float32)
    if kind == "Gather":
        idx, ref = rng.integers(-1, 7, (2, 4)), None
    elif kind == "GatherND":
        idx = rng.integers(0, 6, (3, 4, 1))
    else:
        idx = rng.integers(0, 5, (3, 6, 2))
    idx = idx.astype(np.int32)
    ref = {"Gather": G.gather, "GatherND": G.gather_nd, "GatherElements": G.gather_elements}[kind](params, idx, axis)
    x = Tensor(params.shape, "float", data=torch.from_numpy(params).cuda())
    i = Tensor(idx.shape, "int32", data=torch.from_numpy(idx).cuda())
    y = Tensor((), "float")
    ex = backend.onCreate([x, i], [y], Op(type=kind, extra={"axis": axis}))
    assert ex is not None and ex.onResize([x, i], [y]) == 0 and tuple(y.shape) == ref.shape
    y.data = torch.full(ref.shape, float("nan"), device="cuda")
    assert ex.onExecute([x, i], [y]) == 0
    torch.cuda.synchronize()
    assert np.array_equal(y.data.cpu().numpy(), ref)
