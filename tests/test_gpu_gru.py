"""GRU through the C ABI (include/mnn_b200_gru.h, -m gpu).

Per step against float64: T one-step executes chained through h0, every element of every step's Y_h within the oracle's bound
of one step from the same fp32 inputs (oracle/gru_oracle.py), for both linear_before_reset forms, with NaN guard bands around
every output and x 4 bytes past 16-byte alignment.  A T-step execute equals that chain bit for bit, and a D = 2 execute equals
two D = 1 executes (one on X, one on X reversed with direction 1's weights).  Every launch cell the SM count reaches (oracle
census: LBR, cluster size, resident or streamed R, one or several batch groups, a ragged last group, D, threads per dot product)
is read back through the plan and checked the same way.  One execution resized across cells and back equals a fresh one;
refusals one past each limit keep the previous plan; the first execute after a resize can be captured; a captured graph
replays with new inputs and new weights; repeat executes give the same bits."""
import ctypes as C

import numpy as np
import pytest

from oracle import gru_oracle as G
from tests.test_gpu_conv_f32 import GUARD, ptr

pytestmark = pytest.mark.gpu
NOT_SUPPORT = 2
PLAN_FIELDS = ("lbr", "t", "b", "i", "h", "d", "cs", "groups", "rows", "resident", "smem", "scratch", "launches", "ks")


def glib():
    from mnn_b200 import _capi
    return _capi.gru_lib()


def lib():
    from mnn_b200 import _capi
    return _capi.lib()


def create(backend, lbr):
    h = C.c_void_p()
    assert glib().mnnb200_gru_create(backend.runtime._h, lbr, C.byref(h)) == 0, lib().mnnb200_last_error()
    return h


def plan(h):
    f = (C.c_int * len(PLAN_FIELDS))()
    assert glib().mnnb200_gru_plan(h, f, len(PLAN_FIELDS)) == 0, lib().mnnb200_last_error()
    return dict(zip(PLAN_FIELDS, f))


def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def param_array(ptrs):
    return (C.c_void_p * len(ptrs))(*[p.value if isinstance(p, C.c_void_p) else p for p in ptrs])


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


def execute(backend, h, x, params, h0=None, resize=True, want_y=True, want_yh=True):
    """(Y, Y_h) of one execute on fresh device copies, outputs NaN-poisoned between guards (None where not requested)"""
    T, B, I = x.shape
    D = len(params) // 5
    H = params[3].shape[-1]
    if resize:
        st = glib().mnnb200_gru_resize(h, T, B, I, H, D, int(h0 is not None))
        assert st == 0, lib().mnnb200_last_error()
    xs = Dev(x, 1)
    ps = [Dev(a) for a in params]
    hs = None if h0 is None else Dev(h0)
    y = Dev(np.full((T, D, B, H), np.nan)) if want_y else None
    yh = Dev(np.full((D, B, H), np.nan)) if want_yh else None
    st = glib().mnnb200_gru_execute(h, xs.ptr(), param_array([p.ptr() for p in ps]), None if hs is None else hs.ptr(),
                                    None if y is None else y.ptr(), None if yh is None else yh.ptr())
    assert st == 0, lib().mnnb200_last_error()
    backend.onSync()
    return (None if y is None else y.read((T, D, B, H))), (None if yh is None else yh.read((D, B, H)))


def check_step(lbr, x_t, p, h_prev, yh, what):
    """one direction's step Y_h [B, H] against float64 from the same fp32 inputs, within the step bound"""
    h64, e = G.step_check_bounds(lbr, x_t, p, h_prev)
    assert np.isfinite(yh).all(), f"{what}: non-finite"
    err = np.abs(yh.astype(np.float64) - h64)
    over = err > e
    if over.any():
        i = tuple(np.argwhere(over)[0])
        pytest.fail(f"{what}: {int(over.sum())} of {yh.size} over the bound; first at {i}: got {yh[i]!r}, float64 {h64[i]!r}, "
                    f"|err| {err[i]:.3g} > {e[i]:.3g}")


def chain(backend, h, lbr, x, params, h0, check=True, what=""):
    """T one-step executes of one direction chained through h0: (Y [T, 1, B, H], Y_h), each step checked"""
    hp, ys = h0, []
    for s in range(x.shape[0]):
        y, yh = execute(backend, h, x[s:s + 1], params, hp)
        assert np.array_equal(y[0].view(np.uint32), yh.view(np.uint32)), "Y of the only step differs from Y_h"
        if check:
            check_step(lbr, x[s], params, None if hp is None else hp[0], yh[0], f"{what} step {s}")
        ys.append(y[0])
        hp = yh
    return np.stack(ys), hp


def inputs(rng, T, B, I, H, D, has_h0, scale=None):
    x = rng.standard_normal((T, B, I)).astype(np.float32)
    params = G.random_params(rng, D, I, H, scale)
    h0 = (rng.standard_normal((D, B, H)) * 0.5).astype(np.float32) if has_h0 else None
    return x, params, h0


# (LBR, T, B, I, H, h0, weight scale): B != H, B = 1, T = 1, I != H, H of 1, 3, 33 and 100, B past 8, saturated gates
CASES = [(lbr,) + c for lbr in (0, 1) for c in
         [(6, 3, 20, 33, True, None), (5, 1, 7, 3, False, None), (1, 4, 9, 1, True, None), (4, 5, 16, 33, False, None),
          (4, 2, 12, 17, True, 4.0), (3, 11, 5, 100, True, None)]]


@pytest.mark.parametrize("ci", range(len(CASES)))
def test_per_step_against_float64_and_sequence_equals_chain(backend, ci):
    lbr, T, B, I, H, hh, scale = CASES[ci]
    rng = np.random.default_rng(100 + ci)
    x, params, h0 = inputs(rng, T, B, I, H, 1, hh, scale)
    h = create(backend, lbr)
    try:
        ys, yh_c = chain(backend, h, lbr, x, params, h0, what=str(CASES[ci]))
        y, yh = execute(backend, h, x, params, h0)
        assert plan(h)["launches"] == 3
        assert np.array_equal(y.view(np.uint32), ys.view(np.uint32)), "the T-step execute differs from the chain"
        assert np.array_equal(yh.view(np.uint32), yh_c.view(np.uint32))
        y64, _ = G.run64(lbr, x, params, h0)
        assert np.abs(y - y64).max() <= 1e-3 * max(1.0, np.abs(y64).max())
        # either output alone is the same bits
        y1, _ = execute(backend, h, x, params, h0, resize=False, want_yh=False)
        _, yh1 = execute(backend, h, x, params, h0, resize=False, want_y=False)
        assert np.array_equal(y1.view(np.uint32), y.view(np.uint32)) and np.array_equal(yh1.view(np.uint32), yh.view(np.uint32))
    finally:
        lib().mnnb200_exec_destroy(h)


@pytest.mark.parametrize("lbr", [0, 1])
@pytest.mark.parametrize("hh", [False, True])
def test_bidirectional_equals_two_unidirectional(backend, lbr, hh):
    rng = np.random.default_rng(7 + lbr + 2 * hh)
    T, B, I, H = 5, 3, 10, 24
    x, params, h0 = inputs(rng, T, B, I, H, 2, hh)
    h2, h1 = create(backend, lbr), create(backend, lbr)
    try:
        y, yh = execute(backend, h2, x, params, h0)
        sel = lambda a, d: None if a is None else a[d:d + 1]
        yf, yhf = execute(backend, h1, x, params[:5], sel(h0, 0))
        yb, yhb = execute(backend, h1, x[::-1].copy(), params[5:], sel(h0, 1))
        bits = lambda a: np.ascontiguousarray(a).view(np.uint32)
        assert np.array_equal(bits(y[:, 0]), bits(yf[:, 0])), "direction 0"
        assert np.array_equal(bits(y[:, 1]), bits(yb[::-1, 0])), "direction 1 writes Y at T - 1 - s"
        assert np.array_equal(bits(yh), bits(np.concatenate([yhf, yhb])))
        assert np.array_equal(bits(yh[1]), bits(y[0, 1])), "the backward Y_h is Y[0][1]"
        y64, yh64 = G.run64(lbr, x, params, h0)
        assert np.abs(y - y64).max() <= 1e-3 * max(1.0, np.abs(y64).max())
        assert np.abs(yh - yh64).max() <= 1e-3 * max(1.0, np.abs(yh64).max())
    finally:
        lib().mnnb200_exec_destroy(h2)
        lib().mnnb200_exec_destroy(h1)


def test_census_covers_every_cell_of_this_device():
    cells = G.census(sms())
    assert {k[1] for k in cells} == {1, 2, 4, 8, 16} and {k[2] for k in cells} == {0, 1}
    assert {k[3] for k in cells} == {0, 1} and {k[4] for k in cells} == {0, 1} and {k[5] for k in cells} == {1, 2}
    assert {k[6] for k in cells} == {1, 2, 4, 8} and {k[0] for k in cells} == {0, 1}


@pytest.mark.parametrize("key", sorted(G.census(132)), ids=str)
def test_every_launch_cell(backend, key):
    cells = G.census(sms())
    if key not in cells:
        pytest.skip(f"cell {key} is not reached on {sms()} SMs")
    lbr, B, H, D = cells[key]
    rng = np.random.default_rng(abs(hash(key)) % 2 ** 31)
    I = 7
    x, params, h0 = inputs(rng, 2, B, I, H, D, True)
    h = create(backend, lbr)
    try:
        # one step from h0: every element within the step bound, per direction
        y, yh = execute(backend, h, x[:1], params, h0)
        got = plan(h)
        want = G.choose_plan(lbr, B, H, D, sms())
        assert {k: got[k] for k in ("cs", "groups", "rows", "resident", "smem", "ks")} == \
               {k: want[k] for k in ("cs", "groups", "rows", "resident", "smem", "ks")}, (got, want)
        assert G.cell_of(lbr, B, D, want) == key and got["launches"] == 3
        for d in range(D):
            check_step(lbr, x[0], params[5 * d:5 * d + 5], h0[d], yh[d], f"{key} direction {d}")
        # two steps equal two chained one-step executes (direction 0)
        y2, _ = execute(backend, h, x, params, h0)
        y1, _ = execute(backend, h, x[1:], params, yh)
        assert np.array_equal(y2[0, 0].view(np.uint32), y[0, 0].view(np.uint32))
        assert np.array_equal(y2[1, 0].view(np.uint32), y1[0, 0].view(np.uint32))
    finally:
        lib().mnnb200_exec_destroy(h)


def test_resize_across_cells_and_back_equals_fresh(backend):
    rng = np.random.default_rng(3)
    shapes = [(3, 2, 9, 40, 1), (2, 20, 9, 300, 2), (2, 9, 5, 1000, 1), (3, 2, 9, 40, 1)]
    for lbr in (0, 1):
        h = create(backend, lbr)
        try:
            for T, B, I, H, D in shapes:
                x, params, h0 = inputs(rng, T, B, I, H, D, True)
                y, yh = execute(backend, h, x, params, h0)
                p = plan(h)
                f = create(backend, lbr)
                try:
                    y2, yh2 = execute(backend, f, x, params, h0)
                    assert plan(f) == p
                finally:
                    lib().mnnb200_exec_destroy(f)
                for a, a2 in ((y, y2), (yh, yh2)):
                    assert np.array_equal(a.view(np.uint32), a2.view(np.uint32))
        finally:
            lib().mnnb200_exec_destroy(h)


def test_refusals_keep_the_previous_plan(backend):
    rng = np.random.default_rng(5)
    x, params, h0 = inputs(rng, 3, 2, 6, 16, 1, True)
    h = create(backend, 0)
    try:
        y, _ = execute(backend, h, x, params, h0)
        p = plan(h)
        big = 2 ** 31
        for dims in [(0, 2, 6, 16, 1), (3, 0, 6, 16, 1), (3, 2, 0, 16, 1), (3, 2, 6, 0, 1), (3, 2, 6, 16, 0), (3, 2, 6, 16, 3),
                     (3, 2, 6, G.MAX_HIDDEN + 1, 1), (big // 64, 64, 1, 16, 1), (1, 1, big // 48, 16, 1),
                     (big // (6 * 4096) + 1, 1, 1, 4096, 2), (1, 65535 * 8 + 1, 1, 1, 1)]:
            assert glib().mnnb200_gru_resize(h, *dims, 1) == NOT_SUPPORT, dims
            assert plan(h) == p, dims
        assert glib().mnnb200_gru_resize(h, 3, 2, 6, 16, 1, 2) != 0
        assert plan(h) == p
        y2, _ = execute(backend, h, x, params, h0, resize=False)
        assert np.array_equal(y.view(np.uint32), y2.view(np.uint32))
    finally:
        lib().mnnb200_exec_destroy(h)


def test_first_execute_after_resize_can_be_captured(backend):
    """resize warms the projection MatMul up, so the first execute allocates nothing and replays from a graph"""
    import torch
    rt = backend.runtime._h
    rng = np.random.default_rng(31)
    for lbr in (0, 1):
        x, params, h0 = inputs(rng, 4, 3, 10, 20, 2, True)
        h, g = create(backend, lbr), C.c_void_p()
        try:
            assert glib().mnnb200_gru_resize(h, 4, 3, 10, 20, 2, 1) == 0
            tx, th0 = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (x, h0))
            tp = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in params]
            arr = param_array([ptr(t) for t in tp])
            y, yh = torch.full((4, 2, 3, 20), float("nan"), device="cuda"), torch.full((2, 3, 20), float("nan"), device="cuda")
            backend.onSync()
            assert lib().mnnb200_graph_begin_capture(rt) == 0
            st = glib().mnnb200_gru_execute(h, ptr(tx), arr, ptr(th0), ptr(y), ptr(yh))
            assert lib().mnnb200_graph_end_capture(rt, C.byref(g)) == 0 and st == 0, lib().mnnb200_last_error()
            assert lib().mnnb200_graph_launch(rt, g) == 0
            backend.onSync()
            fresh = create(backend, lbr)
            try:
                want = execute(backend, fresh, x, params, h0)
            finally:
                lib().mnnb200_exec_destroy(fresh)
            assert np.array_equal(y.cpu().numpy().view(np.uint32), want[0].view(np.uint32))
            assert np.array_equal(yh.cpu().numpy().view(np.uint32), want[1].view(np.uint32))
        finally:
            if g.value:
                lib().mnnb200_graph_destroy(g)
            lib().mnnb200_exec_destroy(h)


@pytest.mark.parametrize("lbr", [0, 1])
def test_graph_replay_with_new_inputs_and_weights_and_repeatable(backend, lbr):
    import torch
    rt = backend.runtime._h
    rng = np.random.default_rng(21 + lbr)
    T, B, I, H, D = 6, 4, 12, 40, 2
    sets = [inputs(rng, T, B, I, H, D, True) for _ in range(3)]
    h = create(backend, lbr)
    g = C.c_void_p()
    try:
        x, params, h0 = sets[0]
        assert glib().mnnb200_gru_resize(h, T, B, I, H, D, 1) == 0
        tx, th0 = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (x, h0))
        tp = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in params]
        arr = param_array([ptr(t) for t in tp])
        y, yh = torch.empty((T, D, B, H), device="cuda"), torch.empty((D, B, H), device="cuda")
        call = lambda: glib().mnnb200_gru_execute(h, ptr(tx), arr, ptr(th0), ptr(y), ptr(yh))
        assert call() == 0
        backend.onSync()
        first = y.cpu().numpy().copy()
        assert call() == 0
        backend.onSync()
        assert np.array_equal(first.view(np.uint32), y.cpu().numpy().view(np.uint32)), "two executes differ"
        assert lib().mnnb200_graph_begin_capture(rt) == 0
        assert call() == 0
        assert lib().mnnb200_graph_end_capture(rt, C.byref(g)) == 0, lib().mnnb200_last_error()
        for xs, ps, hs in sets[1:]:
            tx.copy_(torch.from_numpy(xs))
            th0.copy_(torch.from_numpy(hs))
            for t, a in zip(tp, ps):
                t.copy_(torch.from_numpy(a))
            y.fill_(float("nan"))
            backend.onSync()
            assert lib().mnnb200_graph_launch(rt, g) == 0
            backend.onSync()
            replay = y.cpu().numpy().copy()
            assert lib().mnnb200_graph_launch(rt, g) == 0
            backend.onSync()
            assert np.array_equal(replay.view(np.uint32), y.cpu().numpy().view(np.uint32)), "two replays differ"
            fresh = create(backend, lbr)
            try:
                want = execute(backend, fresh, xs, ps, hs)[0]
            finally:
                lib().mnnb200_exec_destroy(fresh)
            assert np.array_equal(replay.view(np.uint32), want.view(np.uint32))
    finally:
        if g.value:
            lib().mnnb200_graph_destroy(g)
        lib().mnnb200_exec_destroy(h)


def test_goldens_within_1e3_of_the_reference_cpu(backend):
    """every recorded golden (the reference CPU's outputs) within 1e-3 of its max |y|, per output; the backward Y_h that the
    reference takes from its scratch (oracle/gru_oracle.py cpu_y_h) against the restatement instead"""
    from tests.golden import make_gru_golden as M
    gold = np.load(M.PATH)
    for name in sorted(M.CASES):
        lbr, keep, n_out, x, params, h0 = M.case_inputs(name)
        h = create(backend, lbr)
        try:
            y, yh = execute(backend, h, x, params, h0)
        finally:
            lib().mnnb200_exec_destroy(h)
        y64, yh64 = G.run64(lbr, x, params, h0)
        tol = lambda ref: 1e-3 * max(1e-6, float(np.abs(ref).max()))
        if keep:
            ref = gold[f"{name}/y"]
            assert np.abs(y - ref).max() <= tol(ref), (name, "y")
        if f"{name}/y_h" in gold:
            ref = gold[f"{name}/y_h"]
            if keep and n_out > 1 and yh.shape[0] == 2:
                assert np.abs(yh[0] - ref[0]).max() <= tol(ref[0]), (name, "y_h forward")
                assert np.abs(yh[1] - yh64[1]).max() <= 1e-3 * max(1.0, float(np.abs(yh64[1]).max())), (name, "y_h backward")
            else:
                assert np.abs(yh - ref).max() <= tol(ref), (name, "y_h")

