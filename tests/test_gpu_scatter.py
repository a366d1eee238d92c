"""ScatterNd and ScatterElements through the C ABI (-m gpu).  Every recorded golden bit for bit (and equal to the numpy
restatement), with NaN guard bands around the output; each launch cell the kernels have, asserted through the plan, with sizes
derived from the SM count: last writer without duplicates, duplicates within one warp, the first and last update in different
CTAs, every update into one slot, the padded-pillar pattern, both copy widths with the output 4 bytes past alignment, the
ordered fold with segments of length 1, a segment spanning sort tiles and CTAs, one segment of 2^20 updates, and every sort
pass count (X just below and just above each digit boundary).  One execution resized across shapes equals a fresh one, and
refusals keep its plan; a captured graph replays with new indices and updates; two executes give identical bits."""
import ctypes as C

import numpy as np
import pytest

from oracle import scatter_oracle as S
from tests.golden import make_scatter_golden as M
from tests.test_gpu_conv_f32 import ptr
from tests.test_gpu_gather import dev

pytestmark = pytest.mark.gpu
NOT_SUPPORT = 2
PLAN_FIELDS = ("mode", "reduction", "n", "s", "r", "x", "path", "passes", "launches", "vec", "init_vec", "grid")
REDS = {None: -1, "add": 0, "sub": 1, "mul": 2}
THREADS, TILE = 256, 2048


def slib():
    from mnn_b200 import _capi
    return _capi.scatter_lib()


def lib():
    from mnn_b200 import _capi
    return _capi.lib()


def ints(v):
    v = list(v)
    return (C.c_int * max(len(v), 1))(*v), len(v)


def create(backend, kind, red=None, with_data=True):
    h = C.c_void_p()
    st = slib().mnnb200_scatter_create(backend.runtime._h, M_KIND[kind], REDS[red], int(with_data), C.byref(h))
    assert st == 0, lib().mnnb200_last_error()
    return h


M_KIND = {"ScatterNd": 0, "ScatterElements": 1}


def resize(h, out, ishape, ushape, axis=0, is_int32=False):
    o, orank = ints(out)
    i, irank = ints(ishape)
    u, urank = ints(ushape)
    return slib().mnnb200_scatter_resize(h, o, orank, i, irank, u, urank, int(axis), int(is_int32))


def plan(h):
    f = (C.c_int * len(PLAN_FIELDS))()
    assert slib().mnnb200_scatter_plan(h, f, len(PLAN_FIELDS)) == 0, lib().mnnb200_last_error()
    return dict(zip(PLAN_FIELDS, f))


def execute(h, idx, upd, data, out_shape, y_off=0, u_off=0):
    """y as the GPU computes it, 4-byte words with -1 (NaN) guard bands checked on both sides"""
    import torch
    _, iv, _ = dev(np.asarray(idx, np.int32))
    _, uv, _ = dev(np.asarray(upd), u_off)
    dv = dev(np.asarray(data), y_off)[1] if data is not None else None
    count = int(np.prod(out_shape))
    yb, yv, start = dev(np.full(count, -7, np.int32), y_off)
    st = slib().mnnb200_scatter_execute(h, ptr(dv) if dv is not None else None, ptr(iv), ptr(uv), ptr(yv))
    assert st == 0, lib().mnnb200_last_error()
    torch.cuda.synchronize()
    host = yb.cpu().numpy()
    assert (host[:start] == -1).all() and (host[start + count:] == -1).all(), "a write outside the output"
    dtype = np.asarray(upd).dtype if data is None else np.asarray(data).dtype
    return host[start:start + count].view(dtype).reshape(out_shape)


def same(y, ref, red):
    if red is None:
        return np.array_equal(y.view(np.uint32), ref.view(np.uint32))
    return np.array_equal(S.canonical(y), S.canonical(ref))


def run_case(backend, kind, out, idx, upd, data=None, red=None, axis=0, y_off=0, u_off=0):
    h = create(backend, kind, red, data is not None)
    try:
        assert resize(h, out, np.shape(idx), np.shape(upd), axis, np.asarray(upd).dtype == np.int32) == 0, lib().mnnb200_last_error()
        y = execute(h, idx, upd, data, out, y_off, u_off)
        ref = S.scatter(kind, out, idx, upd, data, red, axis)
        assert same(y, ref, red), f"{int((S.canonical(y) != S.canonical(ref)).sum())} words differ from the sequential loop"
        return y, plan(h)
    finally:
        lib().mnnb200_exec_destroy(h)


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("name", sorted(M.CASES))
def test_golden_scatters_bit_exact(backend, name):
    c = M.CASES[name]
    idx, upd, data = M.case_inputs(name)
    red = M.reduction(name)
    y, pl = run_case(backend, c["kind"], c["out"], idx, upd, data, red, c.get("axis") or 0)
    shape, sha = M.load()[name]
    assert y.shape == shape and M.digest(y) == sha
    n, _, s, r, _ = S.geometry(c["kind"], c["out"], idx.shape, upd.shape, c.get("axis") or 0)
    assert (pl["mode"], pl["reduction"], pl["n"], pl["s"], pl["r"]) == (M_KIND[c["kind"]], REDS[red], n, s, r)
    assert pl["path"] == (1 if red is None else 2) and pl["grid"] >= 1


def test_copy_paths(backend):
    rng = np.random.default_rng(1)
    idx = rng.permutation(40)[:24].reshape(24, 1).astype(np.int32)
    for s, y_off, u_off, vec in ((768, 0, 0, 16), (768, 1, 0, 4), (768, 0, 1, 4), (3, 0, 0, 4)):
        upd = rng.standard_normal((24, s)).astype(np.float32)
        data = rng.standard_normal((40, s)).astype(np.float32)
        _, pl = run_case(backend, "ScatterNd", (40, s), idx, upd, data, y_off=y_off, u_off=u_off)
        assert pl["path"] == 1 and pl["vec"] == vec and pl["launches"] == 4, (s, y_off, u_off, pl)
        assert pl["init_vec"] == (16 if (40 * s) % 4 == 0 and y_off == 0 else 4), (s, y_off, pl)
    # zero-filled canvas, and an empty update list: y = data only
    _, pl = run_case(backend, "ScatterNd", (40, 4), idx, rng.standard_normal((24, 4)).astype(np.float32))
    assert pl["init_vec"] == 16 and pl["vec"] == 16
    _, pl = run_case(backend, "ScatterNd", (40, 4), np.zeros((0, 1), np.int32), np.zeros((0, 4), np.float32),
                     rng.standard_normal((40, 4)).astype(np.float32))
    assert pl["path"] == 0 and pl["launches"] == 1


def test_index_terms_past_int32_are_skipped(backend):
    # (2^24 + 5) * 256 and -(2^24 - 5) * 256 leave int32: int32 wraparound would land on row 5; the CPU and the kernel skip them
    idx = np.array([[(1 << 24) + 5], [-(1 << 24) + 5], [2]], np.int32)
    upd = np.arange(768, dtype=np.float32).reshape(3, 256)
    data = np.full((16, 256), -1.0, np.float32)
    for red in (None, "add"):
        y, _ = run_case(backend, "ScatterNd", (16, 256), idx, upd, data, red)
        assert (y[5] == -1).all() and (y[2] != -1).all(), red


def cells(sm):
    """name -> (kind, out, idx, upd, data, red): the launch cells, sized from the SM count"""
    rng = np.random.default_rng(sm)
    big = 8 * sm * THREADS + 17                      # more updates than one wave of the capped grid holds
    f = lambda *shape: rng.standard_normal(shape).astype(np.float32)
    out = {}
    out["last_writer_no_duplicates"] = ("ScatterNd", (big + 5, 1), rng.permutation(big + 5)[:big].reshape(-1, 1), f(big, 1), f(big + 5, 1), None)
    out["duplicates_within_one_warp"] = ("ScatterNd", (big // 4 + 1, 2), (np.arange(big) // 4).reshape(-1, 1), f(big, 2), None, None)
    ends = rng.integers(0, 64, big)
    ends[0] = ends[-1] = 5
    out["first_and_last_in_other_ctas"] = ("ScatterNd", (64, 1), ends.reshape(-1, 1), f(big, 1), f(64, 1), None)
    out["every_update_one_slot"] = ("ScatterNd", (8, 3), np.full((big, 1), 6), f(big, 3), f(8, 3), None)
    out["every_update_one_slot_add"] = ("ScatterElements", (8,), np.full(big, 6), f(big), f(8), "add")
    pillars, real = 12000, 7000
    cell = np.zeros(pillars, np.int64)
    cell[:real] = rng.permutation(496 * 432)[:real]
    out["padded_pillars"] = ("ScatterNd", (496 * 432, 64), cell.reshape(-1, 1), np.maximum(f(pillars, 64), 0), None, None)
    out["fold_segments_of_one"] = ("ScatterElements", (big,), rng.permutation(big), f(big), f(big), "add")
    seg = np.concatenate([rng.integers(0, 50, 3 * sm), np.full(3 * TILE + 7, 17), rng.integers(0, 50, 2 * TILE)])
    out["segment_across_tiles_and_ctas"] = ("ScatterElements", (50, 3), np.tile(seg[:, None], (1, 3)), f(seg.size, 3),
                                            f(50, 3), "sub")
    out["one_segment_of_2_20"] = ("ScatterElements", (16,), np.full(1 << 20, 7), f(1 << 20), f(16), "add")
    return out


@pytest.mark.parametrize("name", list(cells(132)))
def test_launch_cells(backend, name):
    sm = sm_count()
    kind, out, idx, upd, data, red = cells(sm)[name]
    y, pl = run_case(backend, kind, out, np.asarray(idx, np.int32), upd, data, red)
    n = int(np.asarray(idx).shape[0])
    if red is None:
        assert pl["path"] == 1 and pl["launches"] == 4
        if name.startswith(("last_writer", "duplicates", "first_and_last")):
            assert pl["grid"] == 8 * sm and n * pl["s"] > pl["grid"] * THREADS, pl
    else:
        assert pl["path"] == 2 and pl["launches"] == 3 + 3 * pl["passes"], pl
    if name == "padded_pillars":
        assert pl["vec"] == 16 and pl["s"] == 64


@pytest.mark.parametrize("x,passes", [(255, 1), (256, 2), (65535, 2), (65536, 3), ((1 << 24) - 1, 3), (1 << 24, 4)])
def test_sort_pass_counts(backend, x, passes):
    rng = np.random.default_rng(x)
    n = 3 * TILE + 100
    idx = rng.integers(0, x, n)
    idx[:40] = x - 1                                  # the top slot, whose digits are all set
    idx[40:80] = 0
    upd = rng.standard_normal(n).astype(np.float32)
    data = rng.standard_normal(x).astype(np.float32)
    _, pl = run_case(backend, "ScatterElements", (x,), idx.astype(np.int32), upd, data, "add")
    assert pl["x"] == x and pl["passes"] == passes and pl["path"] == 2


def test_resize_across_shapes_and_refusals(backend):
    rng = np.random.default_rng(5)
    shapes = [((6, 768), (4, 1), (4, 768)), ((40, 3), (100, 1), (100, 3)), ((5, 4, 3), (10, 2), (10, 3)), ((6, 768), (4, 1), (4, 768))]
    for red in (None, "add"):
        h = create(backend, "ScatterNd", red)
        try:
            for out, ishape, ushape in shapes:
                idx = np.stack([rng.integers(0, out[k], ishape[:-1]) for k in range(ishape[-1])], -1).astype(np.int32)
                upd = rng.standard_normal(ushape).astype(np.float32)
                data = rng.standard_normal(out).astype(np.float32)
                assert resize(h, out, ishape, ushape) == 0
                y = execute(h, idx, upd, data, out)
                assert same(y, S.scatter("ScatterNd", out, idx, upd, data, red), red)
                fresh = create(backend, "ScatterNd", red)
                try:
                    assert resize(fresh, out, ishape, ushape) == 0
                    execute(fresh, idx, upd, data, out)
                    assert plan(fresh) == plan(h)
                finally:
                    lib().mnnb200_exec_destroy(fresh)
            kept = plan(h)
            refusals = [((4, 5, 768), (3, 2), (3, 1, 6, 768), False),  # S = 4608 > R = 768
                        ((6, 768), (4, 1), (3, 768), False),         # fewer than N * S updates
                        ((6, 768), (4, 3), (4, 768), False),         # D past the output's rank
                        ((1,) * 9, (1, 1), (1,), False),             # rank 9
                        ((6, 0), (4, 1), (4, 0), False)]             # empty output
            if red is not None:
                refusals.append(((6, 768), (4, 1), (4, 768), True))  # int32 with a reduction
            for out, ishape, ushape, i32 in refusals:
                assert resize(h, out, ishape, ushape, 0, i32) == NOT_SUPPORT, (out, ishape, ushape)
                assert plan(h) == kept
        finally:
            lib().mnnb200_exec_destroy(h)
    bad = C.c_void_p()
    assert slib().mnnb200_scatter_create(backend.runtime._h, 1, 9, 1, C.byref(bad)) == NOT_SUPPORT   # MAXIMUM


@pytest.mark.parametrize("red", [None, "add"])
def test_graph_replay_with_new_indices_and_repeatable(backend, red):
    import torch
    rt = backend.runtime._h
    rng = np.random.default_rng(11)
    out, n = (300, 16), 5000
    h = create(backend, "ScatterNd", red)
    g = C.c_void_p()
    try:
        assert resize(h, out, (n, 1), (n, 16)) == 0
        sets = [(rng.integers(0, 300, (n, 1)).astype(np.int32), rng.standard_normal((n, 16)).astype(np.float32)) for _ in range(3)]
        data = rng.standard_normal(out).astype(np.float32)
        ib, iv, _ = dev(sets[0][0])
        ub, uv, _ = dev(sets[0][1])
        db, dv, _ = dev(data)
        y = torch.empty(out, dtype=torch.float32, device="cuda")
        call = lambda: slib().mnnb200_scatter_execute(h, ptr(dv), ptr(iv), ptr(uv), C.c_void_p(y.data_ptr()))
        assert call() == 0
        backend.onSync()
        first = y.cpu().numpy().copy()
        assert call() == 0
        backend.onSync()
        assert np.array_equal(first.view(np.uint32), y.cpu().numpy().view(np.uint32)), "two executes differ"
        assert lib().mnnb200_graph_begin_capture(rt) == 0
        assert call() == 0
        assert lib().mnnb200_graph_end_capture(rt, C.byref(g)) == 0, lib().mnnb200_last_error()
        for idx, upd in sets[1:]:
            iv.copy_(torch.from_numpy(idx.view(np.int32).reshape(-1)))
            uv.copy_(torch.from_numpy(upd.view(np.int32).reshape(-1)))
            y.fill_(float("nan"))
            backend.onSync()
            assert lib().mnnb200_graph_launch(rt, g) == 0
            backend.onSync()
            assert same(y.cpu().numpy(), S.scatter("ScatterNd", out, idx, upd, data, red), red)
    finally:
        if g.value:
            lib().mnnb200_graph_destroy(g)
        lib().mnnb200_exec_destroy(h)
