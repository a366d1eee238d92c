"""fp32 BinaryOp, UnaryOp and ArgMax through the C ABI (-m gpu), against numpy.

Every binary op is one round-to-nearest fp32 operation and must equal numpy float32 bit for bit, in all three shape forms
(equal sizes, one-element left side, one-element right side), with and without the fused ReLU.  HARDSWISH, ABS, NEG and
SQUARE are exact as well; the transcendental unary ops come within 1e-5 relative of float64.  ArgMax / ArgMin return the
first extreme index, as CPUArgMax does.  Every output is poisoned before the run."""
import ctypes as C

import numpy as np
import pytest
from scipy import special

pytestmark = pytest.mark.gpu

ADD, SUB, MUL, REALDIV, MINIMUM, MAXIMUM, SQDIFF = 0, 1, 2, 7, 8, 9, 14
BINARY = {
    ADD: lambda a, b: a + b,
    SUB: lambda a, b: a - b,
    MUL: lambda a, b: a * b,
    REALDIV: lambda a, b: a / b,
    MINIMUM: np.minimum,
    MAXIMUM: np.maximum,
    SQDIFF: lambda a, b: (a - b) * (a - b),
}
COUNTS = [1, 3, 4 * 1025 + 3]


def lib():
    from mnn_b200 import _capi
    return _capi.lib()


def dev(a, dtype=np.float32):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, dtype)).cuda()


def poisoned(n, dtype=None):
    import torch
    if dtype is None:
        return torch.full((n,), float("nan"), dtype=torch.float32, device="cuda")
    return torch.full((n,), -7, dtype=dtype, device="cuda")


def ptr(t, offset_elems=0):
    return C.c_void_p(t.data_ptr() + 4 * offset_elems)


def sync(backend):
    assert lib().mnnb200_runtime_sync(backend.runtime._h) == 0


def bits_equal(y, ref):
    y, ref = np.asarray(y, np.float32), np.asarray(ref, np.float32)
    return y.shape == ref.shape and np.array_equal(y, ref)


def binary_operands(rng, op, n):
    a = rng.uniform(-4, 4, n).astype(np.float32)
    b = rng.uniform(-4, 4, n).astype(np.float32)
    if op == REALDIV:   # keep the divisor away from zero
        b = (np.sign(b) * (np.abs(b) + 0.25)).astype(np.float32)
    a[: n // 7] = b[: n // 7]   # equal pairs: MINIMUM / MAXIMUM ties, SUB / SquaredDifference exact zeros
    return a, b


@pytest.mark.parametrize("relu", [0, 1])
@pytest.mark.parametrize("form", ["equal", "scalar_left", "scalar_right"])
@pytest.mark.parametrize("count", COUNTS)
@pytest.mark.parametrize("op", sorted(BINARY))
def test_binary_f32_bit_exact(backend, op, count, form, relu):
    rng = np.random.default_rng(op * 1000 + count)
    a, b = binary_operands(rng, op, count)
    if form == "scalar_left":
        a = a[:1].copy()
    elif form == "scalar_right":
        b = b[:1].copy()
    ref = BINARY[op](a.astype(np.float32), b.astype(np.float32)).astype(np.float32)
    ref = np.broadcast_to(ref, (count,))
    if relu:
        ref = np.maximum(ref, np.float32(0))
    ad, bd, yd = dev(a), dev(b), poisoned(count)
    st = lib().mnnb200_binary_f32(backend.runtime._h, op, ptr(ad), a.size, ptr(bd), b.size, ptr(yd), count, relu)
    assert st == 0, lib().mnnb200_last_error()
    sync(backend)
    assert bits_equal(yd.cpu().numpy(), ref), f"op {op} count {count} {form} relu {relu}"


@pytest.mark.parametrize("op", sorted(BINARY))
def test_binary_f32_misaligned(backend, op):
    """pointers 4 bytes past a 16-byte boundary: the scalar path, same bits"""
    n = 4 * 1025 + 3
    rng = np.random.default_rng(op)
    a, b = binary_operands(rng, op, n + 1)
    ad, bd, yd = dev(a), dev(b), poisoned(n + 1)
    st = lib().mnnb200_binary_f32(backend.runtime._h, op, ptr(ad, 1), n, ptr(bd, 1), n, ptr(yd, 1), n, 0)
    assert st == 0, lib().mnnb200_last_error()
    sync(backend)
    y = yd.cpu().numpy()
    assert np.isnan(y[0]), "wrote before the output pointer"
    assert bits_equal(y[1:], BINARY[op](a[1:], b[1:]))


def test_binary_add_f32_is_binary_f32_add(backend):
    n = 4 * 1025 + 3
    rng = np.random.default_rng(5)
    a, b = binary_operands(rng, ADD, n)
    ad, bd, y1, y2 = dev(a), dev(b), poisoned(n), poisoned(n)
    rt = backend.runtime._h
    assert lib().mnnb200_binary_add_f32(rt, ptr(ad), ptr(bd), ptr(y1), n) == 0
    assert lib().mnnb200_binary_f32(rt, ADD, ptr(ad), n, ptr(bd), n, ptr(y2), n, 0) == 0
    sync(backend)
    assert bits_equal(y1.cpu().numpy(), a + b) and bits_equal(y2.cpu().numpy(), a + b)


def test_binary_f32_scalar_read_on_device_at_replay(backend):
    """a one-element side changed between two replays of one captured graph: the replay sees the new value"""
    rt = backend.runtime._h
    n = 1000
    a = np.linspace(-3, 3, n, dtype=np.float32)
    ad, sd, yd = dev(a), dev(np.array([2.0], np.float32)), poisoned(n)
    g = C.c_void_p()
    sync(backend)
    assert lib().mnnb200_graph_begin_capture(rt) == 0
    assert lib().mnnb200_binary_f32(rt, MUL, ptr(ad), n, ptr(sd), 1, ptr(yd), n, 0) == 0
    assert lib().mnnb200_graph_end_capture(rt, C.byref(g)) == 0, lib().mnnb200_last_error()
    try:
        for s in (2.0, -0.5):
            sd.fill_(s)
            sync(backend)
            assert lib().mnnb200_graph_launch(rt, g) == 0
            sync(backend)
            assert bits_equal(yd.cpu().numpy(), a * np.float32(s))
    finally:
        lib().mnnb200_graph_destroy(g)


def test_binary_f32_unsupported_op(backend):
    ad, yd = dev(np.ones(4, np.float32)), poisoned(4)
    for op in (3, 6, 10, 13, 17, 29, 99):   # DIV, POW, GREATER, FLOORDIV, FLOORMOD, MUL_SILU, not an op
        assert lib().mnnb200_binary_f32(backend.runtime._h, op, ptr(ad), 4, ptr(ad), 4, ptr(yd), 4, 0) == 2
    # a side that is neither count elements nor one
    assert lib().mnnb200_binary_f32(backend.runtime._h, ADD, ptr(ad), 2, ptr(ad), 4, ptr(yd), 4, 0) != 0


# (UnaryOpOperation, float32 reference or None, float64 reference, input domain)
def _hardswish32(x):
    return (x * np.minimum(np.maximum(x + np.float32(3), np.float32(0)), np.float32(6))) / np.float32(6)


UNARY = {
    "ABS": (0, np.abs, np.abs, (-50, 50)),
    "NEG": (1, np.negative, np.negative, (-50, 50)),
    "SQUARE": (4, lambda x: x * x, None, (-50, 50)),
    "SQRT": (5, None, np.sqrt, (0, 100)),
    "RSQRT": (6, None, lambda x: 1 / np.sqrt(x), (1e-3, 100)),
    "EXP": (7, None, np.exp, (-20, 20)),
    "LOG": (8, None, np.log, (1e-4, 100)),
    "RECIPROCAL": (15, None, lambda x: 1 / x, (0.01, 100)),
    "SIGMOID": (29, None, lambda x: 1 / (1 + np.exp(-x)), (-20, 20)),
    "TANH": (30, None, np.tanh, (-10, 10)),
    "HARDSWISH": (31, _hardswish32, None, (-6, 6)),
    "GELU": (32, None, lambda x: 0.5 * x * (1 + np.tanh(0.79788458 * (x + 0.044715 * x ** 3))), (-5, 5)),
    "GELU_STANDARD": (33, None, lambda x: 0.5 * x * (1 + special.erf(x / np.sqrt(2.0))), (-6, 6)),
    "SILU": (34, None, lambda x: x / (1 + np.exp(-x)), (-20, 20)),
}


@pytest.mark.parametrize("name", sorted(UNARY))
def test_unary_f32(backend, name):
    op, ref32, ref64, (lo, hi) = UNARY[name]
    n = 4 * 1025 + 3
    rng = np.random.default_rng(op)
    x = rng.uniform(lo, hi, n).astype(np.float32)
    if lo < 0 < hi:
        x[:5] = np.array([0.0, -3.0, 3.0, -1e-3, 1e-3], np.float32)   # zero, HARDSWISH's kinks, near zero
    xd, yd = dev(x), poisoned(n)
    for off, cnt in ((0, n), (1, n - 1)):   # aligned (float4) and misaligned (scalar) paths
        yd.fill_(float("nan"))
        st = lib().mnnb200_unary_f32(backend.runtime._h, op, ptr(xd, off), ptr(yd, off), cnt)
        assert st == 0, lib().mnnb200_last_error()
        sync(backend)
        y = yd.cpu().numpy()[off:]
        xs = x[off:]
        if ref32 is not None:
            assert bits_equal(y, ref32(xs)), name
        else:
            ref = ref64(xs.astype(np.float64))
            rel = np.abs(y.astype(np.float64) - ref) / np.maximum(np.abs(ref), 1e-30)
            assert float(rel.max()) <= 1e-5, f"{name}: worst relative error {rel.max():.3e} at x = {xs[rel.argmax()]}"


def test_unary_f32_unsupported_op(backend):
    xd, yd = dev(np.ones(4, np.float32)), poisoned(4)
    for op in (2, 3, 9, 10, 16, 22, 23, 25, 99):   # FLOOR, CEIL, SIN, COS, LOG1P, SIGN, ROUND, ERF, not an op
        assert lib().mnnb200_unary_f32(backend.runtime._h, op, ptr(xd), ptr(yd), 4) == 2


def argmax_ref(x, outside, axis, inside, is_min):
    v = x.reshape(outside, axis, inside)
    return (np.argmin(v, axis=1) if is_min else np.argmax(v, axis=1)).astype(np.int32).reshape(-1)   # numpy: first extreme


@pytest.mark.parametrize("is_min", [0, 1])
@pytest.mark.parametrize("view", [(2, 1001, 1), (1, 2, 1001), (3, 7, 5), (64, 33, 1), (4, 1, 9)])
def test_argmax_f32(backend, view, is_min):
    import torch
    outside, axis, inside = view
    rng = np.random.default_rng(axis * 10 + is_min)
    # few distinct values: many ties, the first index must win
    x = rng.integers(-3, 4, outside * axis * inside).astype(np.float32)
    xd, yd = dev(x), poisoned(outside * inside, torch.int32)
    st = lib().mnnb200_argmax_f32(backend.runtime._h, ptr(xd), outside, axis, inside, is_min, ptr(yd))
    assert st == 0, lib().mnnb200_last_error()
    sync(backend)
    assert np.array_equal(yd.cpu().numpy(), argmax_ref(x, outside, axis, inside, is_min))


def test_argmax_f32_all_ties_and_distinct(backend):
    import torch
    rt = backend.runtime._h
    for x, want in ((np.full(1001, 0.25, np.float32), 0), (np.arange(1001, dtype=np.float32)[::-1].copy(), 0),
                    (np.arange(1001, dtype=np.float32), 1000)):
        xd, yd = dev(x), poisoned(1, torch.int32)
        assert lib().mnnb200_argmax_f32(rt, ptr(xd), 1, 1001, 1, 0, ptr(yd)) == 0
        sync(backend)
        assert int(yd.cpu().numpy()[0]) == want
