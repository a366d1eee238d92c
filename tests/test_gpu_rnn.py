"""LSTM and RNN through the C ABI (include/mnn_b200_rnn.h, -m gpu).

Per step against float64: T one-step executes chained through h0 / c0, every element of every step's Y_h / Y_c within the
oracle's bound of one step from the same fp32 inputs (oracle/rnn_oracle.py), with NaN guard bands around every output and x 4
bytes past 16-byte alignment.  A T-step execute equals that chain bit for bit, and a D = 2 execute equals two D = 1 executes (one
on X, one on X reversed with direction 1's weights).  Every launch cell the SM count reaches (oracle census: cluster size,
resident or streamed R, one or several batch groups, a ragged last group, D, threads per dot product, both cells) is read
back through the plan and checked the same way.  One execution resized across cells and back equals a fresh one; refusals one
past each limit keep the previous plan; a captured graph replays with new inputs and new weights; repeat executes give the same
bits."""
import ctypes as C

import numpy as np
import pytest

from oracle import rnn_oracle as R
from tests.test_gpu_conv_f32 import GUARD, ptr

pytestmark = pytest.mark.gpu
NOT_SUPPORT = 2
PLAN_FIELDS = ("cell", "t", "b", "i", "h", "d", "cs", "groups", "rows", "resident", "smem", "scratch", "launches", "ks")


def rlib():
    from mnn_b200 import _capi
    return _capi.rnn_lib()


def lib():
    from mnn_b200 import _capi
    return _capi.lib()


def create(backend, cell):
    h = C.c_void_p()
    assert rlib().mnnb200_rnn_create(backend.runtime._h, cell, C.byref(h)) == 0, lib().mnnb200_last_error()
    return h


def plan(h):
    f = (C.c_int * len(PLAN_FIELDS))()
    assert rlib().mnnb200_rnn_plan(h, f, len(PLAN_FIELDS)) == 0, lib().mnnb200_last_error()
    return dict(zip(PLAN_FIELDS, f))


def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def weights(rng, cell, d, i, h, scale=None):
    g = R.GATES[cell]
    s = scale if scale is not None else 1.0 / np.sqrt(h)
    w = (rng.standard_normal((d, g * h, i)) * s).astype(np.float32)
    r = (rng.standard_normal((d, g * h, h)) * s).astype(np.float32)
    b = (rng.standard_normal((d, g * h)) * 0.5).astype(np.float32)
    return w, r, b


class Dev:
    """a device copy of x between NaN guards, `shift` floats past GUARD (GUARD * 4 bytes is 4 past 16-byte alignment)"""

    def __init__(self, a, shift=0):
        import torch
        a = np.ascontiguousarray(a, np.float32)
        self.n, self.start = a.size, GUARD + shift
        self.buf = torch.full((a.size + 2 * GUARD + shift,), float("nan"), dtype=torch.float32, device="cuda")
        self.view = self.buf[self.start:self.start + self.n]
        self.view.copy_(torch.from_numpy(a.reshape(-1)))

    def ptr(self):
        return ptr(self.view)

    def read(self, shape):
        host = self.buf.cpu().numpy()
        assert np.isnan(host[:self.start]).all() and np.isnan(host[self.start + self.n:]).all(), "a write outside the tensor"
        return host[self.start:self.start + self.n].reshape(shape)


def execute(backend, h, cell, x, w, r, b, h0=None, c0=None, resize=True):
    """(Y, Y_h, Y_c) of one execute on fresh device copies, outputs NaN-poisoned between guards"""
    T, B, I = x.shape
    D, _, H = r.shape
    if resize:
        st = rlib().mnnb200_rnn_resize(h, T, B, I, H, D, int(h0 is not None), int(c0 is not None))
        assert st == 0, lib().mnnb200_last_error()
    xs = Dev(x, 1)
    ins = [Dev(a) for a in (w, r, b)]
    st0 = [None if a is None else Dev(a) for a in (h0, c0)]
    y, yh = Dev(np.full((T, D, B, H), np.nan)), Dev(np.full((D, B, H), np.nan))
    yc = Dev(np.full((D, B, H), np.nan)) if cell == 0 else None
    st = rlib().mnnb200_rnn_execute(h, xs.ptr(), *[a.ptr() for a in ins], *[None if a is None else a.ptr() for a in st0],
                                    y.ptr(), yh.ptr(), None if yc is None else yc.ptr())
    assert st == 0, lib().mnnb200_last_error()
    backend.onSync()
    return y.read((T, D, B, H)), yh.read((D, B, H)), None if yc is None else yc.read((D, B, H))


def check_step(cell, x_t, w, r, b, h_prev, c_prev, yh, yc, what):
    """one D = 1 step's Y_h / Y_c against float64 from the same fp32 inputs, within the step bound"""
    gate, gabs = R.gates64(x_t, w[0], b[0])
    h64, c64, eh, ec = R.step_check_bounds(cell, gate, gabs, x_t.shape[1], b[0], r[0], h_prev, c_prev)
    for got, ref, e, name in ((yh[0], h64, eh, "Y_h"), (None if yc is None else yc[0], c64, ec, "Y_c")):
        if got is None:
            continue
        assert np.isfinite(got).all(), f"{what} {name}: non-finite"
        err = np.abs(got.astype(np.float64) - ref)
        over = err > e
        if over.any():
            i = tuple(np.argwhere(over)[0])
            pytest.fail(f"{what} {name}: {int(over.sum())} of {got.size} over the bound; first at {i}: got {got[i]!r}, "
                        f"float64 {ref[i]!r}, |err| {err[i]:.3g} > {e[i]:.3g}")


def chain(backend, h, cell, x, w, r, b, h0, c0, check=True, what=""):
    """T one-step executes of one direction chained through h0 / c0: (Y [T, 1, B, H], Y_h, Y_c), each step checked"""
    hp, cp = h0, c0
    ys = []
    for s in range(x.shape[0]):
        y, yh, yc = execute(backend, h, cell, x[s:s + 1], w, r, b, hp, cp if cell == 0 else None)
        assert np.array_equal(y[0].view(np.uint32), yh.view(np.uint32)), "Y of the only step differs from Y_h"
        if check:
            check_step(cell, x[s], w, r, b, None if hp is None else hp[0], None if (cell == 1 or cp is None) else cp[0],
                       yh, yc, f"{what} step {s}")
        ys.append(y[0])
        hp, cp = yh, (yc if cell == 0 else None)
    return np.stack(ys), hp, cp


INIT = {"none": (False, False), "h0": (True, False), "h0c0": (True, True)}
# (cell, T, B, I, H, init, weight scale): B != H, B = 1, T = 1, I != H, H of 1, 3 and 33, saturated gates
CASES = [(0, 6, 3, 20, 33, "h0c0", None), (0, 5, 1, 7, 3, "none", None), (0, 1, 4, 9, 1, "h0c0", None),
         (0, 4, 5, 16, 33, "h0", None), (0, 4, 2, 12, 17, "h0c0", 4.0), (1, 6, 3, 20, 33, "h0", None),
         (1, 5, 1, 7, 3, "none", None), (1, 3, 2, 8, 1, "h0", None), (1, 4, 3, 12, 17, "h0", 4.0)]


def inputs(rng, cell, T, B, I, H, D, init, scale):
    x = rng.standard_normal((T, B, I)).astype(np.float32)
    w, r, b = weights(rng, cell, D, I, H, scale)
    hh, hc = INIT[init]
    h0 = rng.standard_normal((D, B, H)).astype(np.float32) * 0.5 if hh else None
    c0 = rng.standard_normal((D, B, H)).astype(np.float32) if (hc and cell == 0) else None
    return x, w, r, b, h0, c0


@pytest.mark.parametrize("ci", range(len(CASES)))
def test_per_step_against_float64_and_sequence_equals_chain(backend, ci):
    cell, T, B, I, H, init, scale = CASES[ci]
    rng = np.random.default_rng(100 + ci)
    x, w, r, b, h0, c0 = inputs(rng, cell, T, B, I, H, 1, init, scale)
    h = create(backend, cell)
    try:
        ys, yh_c, yc_c = chain(backend, h, cell, x, w, r, b, h0, c0, what=str(CASES[ci]))
        y, yh, yc = execute(backend, h, cell, x, w, r, b, h0, c0)
        assert plan(h)["launches"] == 1
        assert np.array_equal(y.view(np.uint32), ys.view(np.uint32)), "the T-step execute differs from the chain"
        assert np.array_equal(yh.view(np.uint32), yh_c.view(np.uint32))
        if cell == 0:
            assert np.array_equal(yc.view(np.uint32), yc_c.view(np.uint32))
        y64, _, _ = R.run64(cell, x, w, r, b, h0, c0)
        assert np.abs(y - y64).max() <= 1e-3 * max(1.0, np.abs(y64).max())
    finally:
        lib().mnnb200_exec_destroy(h)


@pytest.mark.parametrize("cell", [0, 1])
@pytest.mark.parametrize("init", ["none", "h0c0"])
def test_bidirectional_equals_two_unidirectional(backend, cell, init):
    rng = np.random.default_rng(7 + cell)
    T, B, I, H = 5, 3, 10, 24
    x, w, r, b, h0, c0 = inputs(rng, cell, T, B, I, H, 2, init, None)
    h2, h1 = create(backend, cell), create(backend, cell)
    try:
        y, yh, yc = execute(backend, h2, cell, x, w, r, b, h0, c0)
        sel = lambda a, d: None if a is None else a[d:d + 1]
        yf, yhf, ycf = execute(backend, h1, cell, x, w[:1], r[:1], b[:1], sel(h0, 0), sel(c0, 0))
        yb, yhb, ycb = execute(backend, h1, cell, x[::-1].copy(), w[1:], r[1:], b[1:], sel(h0, 1), sel(c0, 1))
        bits = lambda a: np.ascontiguousarray(a).view(np.uint32)
        assert np.array_equal(bits(y[:, 0]), bits(yf[:, 0])), "direction 0"
        assert np.array_equal(bits(y[:, 1]), bits(yb[::-1, 0])), "direction 1 writes Y at T - 1 - s"
        assert np.array_equal(bits(yh), bits(np.concatenate([yhf, yhb])))
        if cell == 0:
            assert np.array_equal(bits(yc), bits(np.concatenate([ycf, ycb])))
        y64, yh64, _ = R.run64(cell, x, w, r, b, h0, c0)
        assert np.abs(y - y64).max() <= 1e-3 * max(1.0, np.abs(y64).max())
    finally:
        lib().mnnb200_exec_destroy(h2)
        lib().mnnb200_exec_destroy(h1)


def test_census_covers_every_cell_of_this_device():
    cells = R.census(sms())
    assert {k[1] for k in cells} == {1, 2, 4, 8, 16} and {k[2] for k in cells} == {0, 1}
    assert {k[3] for k in cells} == {0, 1} and {k[4] for k in cells} == {0, 1} and {k[5] for k in cells} == {1, 2}
    assert {k[6] for k in cells} == {1, 2, 4, 8}


@pytest.mark.parametrize("key", sorted(R.census(132)), ids=str)
def test_every_launch_cell(backend, key):
    cells = R.census(sms())
    if key not in cells:
        pytest.skip(f"cell {key} is not reached on {sms()} SMs")
    cell, B, H, D = cells[key]
    rng = np.random.default_rng(abs(hash(key)) % 2 ** 31)
    I = 7
    x, w, r, b, h0, c0 = inputs(rng, cell, 2, B, I, H, D, "h0c0", None)
    h = create(backend, cell)
    try:
        # one step with states: every element within the step bound, per direction
        y, yh, yc = execute(backend, h, cell, x[:1], w, r, b, h0, c0)
        got = plan(h)
        want = R.choose_plan(cell, B, H, D, sms())
        assert {k: got[k] for k in ("cs", "groups", "rows", "resident", "smem", "ks")} == \
               {k: want[k] for k in ("cs", "groups", "rows", "resident", "smem", "ks")}, (got, want)
        assert R.cell_of(cell, B, D, want) == key and got["launches"] == 1
        for d in range(D):
            check_step(cell, x[0], w[d:d + 1], r[d:d + 1], b[d:d + 1], h0[d], None if c0 is None else c0[d], yh[d:d + 1],
                       None if yc is None else yc[d:d + 1], f"{key} direction {d}")
        # two steps equal two chained one-step executes (direction 0)
        y2, _, _ = execute(backend, h, cell, x, w, r, b, h0, c0)
        yc0 = None if yc is None else yc
        y1, yh1, yc1 = execute(backend, h, cell, x[1:], w, r, b, yh, yc0)
        assert np.array_equal(y2[0, 0].view(np.uint32), y[0, 0].view(np.uint32))
        assert np.array_equal(y2[1, 0].view(np.uint32), y1[0, 0].view(np.uint32))
    finally:
        lib().mnnb200_exec_destroy(h)


def test_resize_across_cells_and_back_equals_fresh(backend):
    rng = np.random.default_rng(3)
    shapes = [(0, 3, 2, 9, 40, 1), (0, 2, 20, 9, 300, 2), (0, 2, 9, 5, 1000, 1), (0, 3, 2, 9, 40, 1)]
    h = create(backend, 0)
    try:
        for cell, T, B, I, H, D in shapes:
            x, w, r, b, h0, c0 = inputs(rng, cell, T, B, I, H, D, "h0c0", None)
            y, yh, yc = execute(backend, h, cell, x, w, r, b, h0, c0)
            p = plan(h)
            f = create(backend, cell)
            try:
                y2, yh2, yc2 = execute(backend, f, cell, x, w, r, b, h0, c0)
                assert plan(f) == p
            finally:
                lib().mnnb200_exec_destroy(f)
            for a, a2 in ((y, y2), (yh, yh2), (yc, yc2)):
                assert np.array_equal(a.view(np.uint32), a2.view(np.uint32))
    finally:
        lib().mnnb200_exec_destroy(h)


def test_refusals_keep_the_previous_plan(backend):
    rng = np.random.default_rng(5)
    x, w, r, b, h0, c0 = inputs(rng, 0, 3, 2, 6, 16, 1, "h0c0", None)
    h = create(backend, 0)
    try:
        y, _, _ = execute(backend, h, 0, x, w, r, b, h0, c0)
        p = plan(h)
        big = 2 ** 31
        for dims in [(0, 2, 6, 16, 1), (3, 0, 6, 16, 1), (3, 2, 0, 16, 1), (3, 2, 6, 0, 1), (3, 2, 6, 16, 0), (3, 2, 6, 16, 3),
                     (3, 2, 6, R.MAX_HIDDEN + 1, 1), (big // 64, 64, 1, 16, 1), (1, 1, big // 64, 16, 1),
                     (big // (8 * 4096) + 1, 1, 1, 4096, 2), (1, 65535 * 8 + 1, 1, 1, 1)]:
            assert rlib().mnnb200_rnn_resize(h, *dims, 1, 1) == NOT_SUPPORT, dims
            assert plan(h) == p, dims
        y2, _, _ = execute(backend, h, 0, x, w, r, b, h0, c0, resize=False)
        assert np.array_equal(y.view(np.uint32), y2.view(np.uint32))
        assert rlib().mnnb200_rnn_resize(h, 3, 2, 6, 16, 1, 1, 2) != 0
        assert plan(h) == p
    finally:
        lib().mnnb200_exec_destroy(h)


@pytest.mark.parametrize("cell", [0, 1])
def test_graph_replay_with_new_inputs_and_weights_and_repeatable(backend, cell):
    import torch
    rt = backend.runtime._h
    rng = np.random.default_rng(21 + cell)
    T, B, I, H, D = 6, 4, 12, 40, 2
    sets = [inputs(rng, cell, T, B, I, H, D, "h0c0", None) for _ in range(3)]
    h = create(backend, cell)
    g = C.c_void_p()
    try:
        x, w, r, b, h0, c0 = sets[0]
        assert rlib().mnnb200_rnn_resize(h, T, B, I, H, D, 1, int(cell == 0)) == 0
        tens = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (x, w, r, b, h0)] + \
               [torch.from_numpy(c0).cuda() if cell == 0 else None]
        y = torch.empty((T, D, B, H), device="cuda")
        yh, yc = torch.empty((D, B, H), device="cuda"), torch.empty((D, B, H), device="cuda")
        call = lambda: rlib().mnnb200_rnn_execute(h, *[None if t is None else ptr(t) for t in tens], ptr(y), ptr(yh), ptr(yc))
        assert call() == 0
        backend.onSync()
        first = y.cpu().numpy().copy()
        assert call() == 0
        backend.onSync()
        assert np.array_equal(first.view(np.uint32), y.cpu().numpy().view(np.uint32)), "two executes differ"
        assert lib().mnnb200_graph_begin_capture(rt) == 0
        assert call() == 0
        assert lib().mnnb200_graph_end_capture(rt, C.byref(g)) == 0, lib().mnnb200_last_error()
        for s in sets[1:]:
            for t, a in zip(tens, s):
                if t is not None:
                    t.copy_(torch.from_numpy(np.ascontiguousarray(a)))
            y.fill_(float("nan"))
            backend.onSync()
            assert lib().mnnb200_graph_launch(rt, g) == 0
            backend.onSync()
            fresh = create(backend, cell)
            try:
                want = execute(backend, fresh, cell, *s[:5], s[5] if cell == 0 else None)[0]
            finally:
                lib().mnnb200_exec_destroy(fresh)
            assert np.array_equal(y.cpu().numpy().view(np.uint32), want.view(np.uint32))
    finally:
        if g.value:
            lib().mnnb200_graph_destroy(g)
        lib().mnnb200_exec_destroy(h)


def test_goldens_within_1e3_of_the_reference_cpu(backend):
    """every recorded golden (the reference CPU's outputs) within 1e-3 of its max |y|, per output"""
    from tests.golden import make_rnn_golden as M
    gold = np.load(M.PATH)
    for name in sorted(M.CASES):
        cell, x, w, r, b, h0, c0 = M.case_inputs(name)
        h = create(backend, cell)
        try:
            got = execute(backend, h, cell, x, w, r, b, h0, c0)
        finally:
            lib().mnnb200_exec_destroy(h)
        for k, y in zip(("y", "y_h", "y_c"), got):
            if y is None:
                continue
            ref = gold[f"{name}/{k}"]
            assert np.abs(y - ref).max() <= 1e-3 * max(1e-6, float(np.abs(ref).max())), (name, k)


def test_first_execute_after_resize_can_be_captured(backend):
    """resize warms the projection MatMul up, so the first execute allocates nothing and replays from a graph"""
    import torch
    rt = backend.runtime._h
    rng = np.random.default_rng(31)
    x, w, r, b, h0, c0 = inputs(rng, 0, 4, 3, 10, 20, 1, "h0c0", None)
    h, g = create(backend, 0), C.c_void_p()
    try:
        assert rlib().mnnb200_rnn_resize(h, 4, 3, 10, 20, 1, 1, 1) == 0
        tens = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (x, w, r, b, h0, c0)]
        y, yh, yc = (torch.full(s, float("nan"), device="cuda") for s in ((4, 1, 3, 20), (1, 3, 20), (1, 3, 20)))
        backend.onSync()
        assert lib().mnnb200_graph_begin_capture(rt) == 0
        st = rlib().mnnb200_rnn_execute(h, *[ptr(t) for t in tens], ptr(y), ptr(yh), ptr(yc))
        assert lib().mnnb200_graph_end_capture(rt, C.byref(g)) == 0 and st == 0, lib().mnnb200_last_error()
        assert lib().mnnb200_graph_launch(rt, g) == 0
        backend.onSync()
        fresh = create(backend, 0)
        try:
            want = execute(backend, fresh, 0, x, w, r, b, h0, c0)[0]
        finally:
            lib().mnnb200_exec_destroy(fresh)
        assert np.array_equal(y.cpu().numpy().view(np.uint32), want.view(np.uint32))
    finally:
        if g.value:
            lib().mnnb200_graph_destroy(g)
        lib().mnnb200_exec_destroy(h)


def test_recurrence_kernels_compile_without_spills(tmp_path):
    import os
    import subprocess
    from mnn_b200 import build as B
    src = os.path.join(B.CSRC, "rnn.cu")
    out = subprocess.run([os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc"), "-c", src, "-o", str(tmp_path / "rnn.o"),
                          "-Xptxas", "-v"] + B.NVCC_FLAGS, capture_output=True, text=True, check=True).stderr
    spills = [l for l in out.splitlines() if "spill" in l and not l.strip().startswith("0 bytes stack frame, 0 bytes spill")]
    assert "rnn_recur_f32_kernel" in out and not spills, spills
