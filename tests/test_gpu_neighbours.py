"""The kernels around the int8 conv path (-m gpu), each against a plain reference of the same operation:
int8 add, average pool between int8 tensors and int8 softmax (NHWC16), and the fp32 pool / ReLU / reduction / raster /
transpose kernels.  Every int8 output is poisoned with 77 before the run and every fp32 output with NaN, and the NHWC16
channel padding of an int8 output must come back zero."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as O
from tests.test_pool import POOL_CONFIGS, pool_input, session_attrs

pytestmark = pytest.mark.gpu
U = 2.0 ** -24          # unit roundoff of fp32 (round to nearest)


def up16(c):
    return (c + 15) // 16 * 16


def lib():
    from mnn_b200 import _capi
    return _capi.lib()


def int8_in(backend, x, q):
    from mnn_b200.backend import Tensor
    t = backend.onAcquire(Tensor(x.shape, "int8", q))
    backend.onCopyBuffer(x, t)
    return t


def int8_out(backend, t):
    """allocate t (its shape set by onResize) and poison it, padding included"""
    backend.onAcquire(t)
    t.data.fill_(77)
    return t


def int8_result(backend, t):
    """NHWC16 device tensor -> NCHW int8; asserts the channel padding is zero"""
    backend.onSync()
    raw = t.data.cpu().numpy()
    c = t.shape[1]
    assert not raw[..., c:].any(), "NHWC16 channel padding not zero"
    return np.ascontiguousarray(raw[..., :c].transpose(0, 3, 1, 2))


def f32_dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def nan_dev(shape):
    import torch
    return torch.full(shape, float("nan"), dtype=torch.float32, device="cuda")


def bits_equal(y, ref):
    return y.shape == ref.shape and np.array_equal(np.ascontiguousarray(y, np.float32).view(np.uint32),
                                                   np.ascontiguousarray(ref, np.float32).view(np.uint32))


# ---------------------------------------------------------------------------------------------------------------------
# int8 add: bit-exact vs O.binary_add_int8
# ---------------------------------------------------------------------------------------------------------------------
def run_add(backend, x0, q0, x1, q1, qo):
    from mnn_b200.backend import Op, Tensor
    a, b = int8_in(backend, x0, q0), int8_in(backend, x1, q1)
    y = Tensor(x0.shape, "int8", qo)
    ex = backend.onCreate([a, b], [y], Op(type="BinaryAddInt8"))
    assert ex is not None and ex.onResize([a, b], [y]) == 0
    int8_out(backend, y)
    assert ex.onExecute([a, b], [y]) == 0
    got = int8_result(backend, y)
    ref = O.binary_add_int8(x0, (q0.scale, q0.zero), x1, (q1.scale, q1.zero), (qo.scale, qo.zero, qo.min, qo.max))
    return got, ref


@pytest.mark.parametrize("c", [1, 15, 16, 17, 130])
def test_add_int8_vs_oracle(backend, c):
    from mnn_b200.backend import QuantAttr
    rng = np.random.default_rng(c)
    x0 = rng.integers(-128, 128, (2, c, 5, 7)).astype(np.int8)
    x1 = rng.integers(-128, 128, (2, c, 5, 7)).astype(np.int8)
    got, ref = run_add(backend, x0, QuantAttr(0.031, 3), x1, QuantAttr(0.047, -5), QuantAttr(0.06, -2, -127, 127))
    assert np.array_equal(got, ref)


def test_add_int8_half_ties(backend):
    """s0 = s1 = 0.5, s_out = 1: every odd q0 + q1 lands exactly on a .5 tie, which roundf takes away from zero"""
    from mnn_b200.backend import QuantAttr
    rng = np.random.default_rng(5)
    x0 = rng.integers(-128, 128, (3, 33, 4, 6)).astype(np.int8)
    x1 = rng.integers(-128, 128, (3, 33, 4, 6)).astype(np.int8)
    got, ref = run_add(backend, x0, QuantAttr(0.5, 0), x1, QuantAttr(0.5, 0), QuantAttr(1.0, 0, -128, 127))
    ties = (x0.astype(int) + x1.astype(int)) % 2 == 1
    assert ties.mean() > 0.4
    assert np.array_equal(got, ref)


def test_add_int8_saturation_and_large(backend):
    """~9 % of the outputs saturate; 8 x 130 x 112 x 112 (1.6 M 16-byte chunks) spans many waves of the grid.  (The grid
    covers the work up to 2^31 - 1 blocks, so its grid-stride loop does not wrap at any size a tensor can have.)"""
    from mnn_b200.backend import QuantAttr
    rng = np.random.default_rng(9)
    x0 = rng.integers(-128, 128, (8, 130, 112, 112)).astype(np.int8)
    x1 = rng.integers(-128, 128, (8, 130, 112, 112)).astype(np.int8)
    qo = QuantAttr(0.07, 1, -128, 127)
    got, ref = run_add(backend, x0, QuantAttr(0.05, 0), x1, QuantAttr(0.05, 0), qo)
    sat = np.mean((ref == -128) | (ref == 127))
    assert 0.02 < sat < 0.12, sat
    assert np.array_equal(got, ref)


# ---------------------------------------------------------------------------------------------------------------------
# average pool between int8 tensors (AvgPoolInt8Execution): bit-exact vs O.avgpool_int8_via_float on both kernels
# ---------------------------------------------------------------------------------------------------------------------
AVG_SWITCH = 64 * 1024    # launch_avgpool_int8_via_float: fewer 16-channel work items -> one channel per thread


def run_avgpool(backend, x, attrs, qi, qo):
    from mnn_b200.backend import Op, Tensor
    xt = int8_in(backend, x, qi)
    y = Tensor((1, 1, 1, 1), "int8", qo)
    ex = backend.onCreate([xt], [y], Op(type="AvgPoolInt8", extra=attrs))
    assert ex is not None and ex.onResize([xt], [y]) == 0
    int8_out(backend, y)
    assert ex.onExecute([xt], [y]) == 0
    return int8_result(backend, y)


def resolve(cfg):
    return O.pool_resolve(cfg["ih"], cfg["iw"], cfg["kernel"], cfg["stride"], cfg["pad"], cfg["pads"], cfg["pad_type"],
                          cfg["ceil_model"], cfg["is_global"])


def avgpool_oracle(x, cfg, qi, qo):
    oh, ow, k, s, p, pt = resolve(cfg)
    return O.avgpool_int8_via_float(x, k, s, p, (qi.scale, qi.zero), (qo.scale, qo.zero, qo.min, qo.max), pt,
                                    cfg["count_type"], out=(oh, ow))


@pytest.mark.parametrize("side", ["1ch", "16ch"])
@pytest.mark.parametrize("ci", range(len(POOL_CONFIGS)))
def test_avgpool_int8_vs_oracle(backend, ci, side):
    from mnn_b200.backend import QuantAttr
    cfg = POOL_CONFIGS[ci]
    c = 40
    rng = np.random.default_rng(1000 + ci)
    oh, ow = resolve(cfg)[:2]
    per_image = oh * ow * (up16(c) // 16)
    n = 2 if side == "1ch" else -(-AVG_SWITCH * 11 // 10 // per_image)
    assert (n * per_image < AVG_SWITCH) == (side == "1ch")
    if side == "1ch":
        qi, qo = QuantAttr(0.043, 3), QuantAttr(0.031, -4, -127, 127)
        x = rng.integers(-128, 128, (n, c, cfg["ih"], cfg["iw"])).astype(np.int8)
    else:
        # s_in = 0.5, s_out = 1/9: a 3x3 window's exact mean / s_out is a multiple of 0.5, so the fp32 operation order
        # decides the rounding of every odd sum
        qi, qo = QuantAttr(0.5, 0), QuantAttr(np.float32(1 / 9), 0, -128, 127)
        x = rng.integers(-25, 26, (n, c, cfg["ih"], cfg["iw"])).astype(np.int8)
    got = run_avgpool(backend, x, session_attrs(cfg), qi, qo)
    ref = avgpool_oracle(x, cfg, qi, qo)
    assert got.shape == ref.shape
    assert np.array_equal(got, ref), f"{np.count_nonzero(got != ref)} of {ref.size} differ"


@pytest.mark.parametrize("batch", [32])
def test_avgpool_int8_mobilenet_global(backend, batch):
    from mnn_b200.backend import QuantAttr
    rng = np.random.default_rng(7)
    x = rng.integers(-128, 128, (batch, 1280, 7, 7)).astype(np.int8)
    cfg = POOL_CONFIGS[19]
    assert cfg["is_global"] and (cfg["ih"], cfg["iw"]) == (7, 7)
    qi, qo = QuantAttr(0.0235, -128), QuantAttr(0.0118, -128, -128, 127)
    got = run_avgpool(backend, x, session_attrs(cfg), qi, qo)
    assert np.array_equal(got, avgpool_oracle(x, cfg, qi, qo))


# ---------------------------------------------------------------------------------------------------------------------
# softmax over the channel axis of an int8 [rows][c] tensor
# ---------------------------------------------------------------------------------------------------------------------
def softmax_rows(rng, c):
    """(x, s_in) pairs: random logits, a constant row, one dominant logit, and logits spread wide enough that exp()
    overflows fp32 without the max subtraction"""
    rows = [(rng.integers(-128, 128, (4, c)), 0.05), (np.full((2, c), 37), 0.05)]
    dom = np.full((2, c), -128)
    dom[0, c // 3] = 127
    dom[1, c - 1] = 127
    rows.append((dom, 0.1))
    rows.append((rng.integers(-128, 128, (4, c)), 0.9))
    return [(x.astype(np.int8), s) for x, s in rows]


def softmax_tolerance(t, s_out, c):
    """Bound on |q - (p64 / s_out + z_out)| (before the clamp, which is 1-Lipschitz) from the kernel's fp32 steps, with
    u = 2^-24 and t the dequantised logits (exact fp32 inputs of both computations):
      d = fl(t - max)          relative error u, i.e. an absolute error <= u|d| in the argument of exp
      e = expf(d)              <= 2 ulp (CUDA expf) -> relative 2^-22, plus e^(u|d|) - 1 ~ u|d| from the argument
      S = sum of c terms e     any summation order: relative <= (c - 1) u (all terms positive) on top of the terms' own error
      r = fl(1 / S), p = fl(e r)            u each
      f = fma(p, 1/s_out, z)   fl(1 / s_out) and the fma: u each relative to p / s_out, plus u * 256 absolute (|f| < 256)
      q = trunc(f +- 0.5)      the round: 0.5, plus the fp32 add of 0.5: 2^-17
    The relative terms are summed with a 1 % allowance for their products."""
    d = np.abs(t - t.max(axis=1, keepdims=True))
    e_rel = d * U + 2.0 ** -22
    rho = e_rel + e_rel.max(axis=1, keepdims=True) + (c - 1) * U + 2 * U + 2 * U
    return 0.5 + 1.01 * rho / s_out + 256 * U + 2.0 ** -17


@pytest.mark.parametrize("c", [1, 2, 31, 255, 256, 257, 1001, 4000])
def test_softmax_int8(backend, c):
    from mnn_b200.backend import Op, QuantAttr, Tensor
    rng = np.random.default_rng(c)
    qo = QuantAttr(1 / 256, -128, -128, 127)
    for x, s_in in softmax_rows(rng, c):
        qi = QuantAttr(s_in, 3)
        rows = x.shape[0]
        xt = int8_in(backend, x.reshape(rows, c, 1, 1), qi)
        y = Tensor((rows, c, 1, 1), "int8", qo)
        ex = backend.onCreate([xt], [y], Op(type="SoftmaxInt8"))
        int8_out(backend, y)
        assert ex.onExecute([xt], [y]) == 0
        got = int8_result(backend, y).reshape(rows, c).astype(np.int64)
        ref = O.softmax_int8(x, (qi.scale, qi.zero), (qo.scale, qo.zero, qo.min, qo.max)).astype(np.int64)
        assert np.abs(got - ref).max() <= 1, (s_in, np.abs(got - ref).max())
        t = O.int8_to_float(x, qi.scale, qi.zero).astype(np.float64)
        ex64 = np.exp(t - t.max(axis=1, keepdims=True))
        p64 = ex64 / ex64.sum(axis=1, keepdims=True)
        v64 = np.clip(p64 / np.float64(np.float32(qo.scale)) + qo.zero, qo.min, qo.max)
        tol = softmax_tolerance(t, np.float64(np.float32(qo.scale)), c)
        err = np.abs(got - v64)
        assert (err <= tol).all(), (s_in, float((err - tol).max()))


# ---------------------------------------------------------------------------------------------------------------------
# fp32 pool: bit-exact vs O.pool_f32 (the restatement pinned on the reference in tests/test_pool.py)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("is_avg", [True, False], ids=["ave", "max"])
@pytest.mark.parametrize("ci", range(len(POOL_CONFIGS)))
def test_pool_f32_vs_oracle(backend, ci, is_avg):
    cfg = POOL_CONFIGS[ci]
    x = pool_input(np.random.default_rng(2000 + ci), 3, 19, cfg)
    n, c, ih, iw = x.shape
    oh, ow, (kh, kw), (sh, sw), (ph, pw), pt = resolve(cfg)
    xd, yd = f32_dev(x), nan_dev((n, c, oh, ow))
    assert lib().mnnb200_pool_f32(backend.runtime._h, C.c_void_p(xd.data_ptr()), n, c, ih, iw, kh, kw, sh, sw, ph, pw, pt,
                                  cfg["count_type"], int(is_avg), C.c_void_p(yd.data_ptr()), oh, ow) == 0
    backend.onSync()
    ref = O.pool_f32(x, is_avg, **{k: cfg[k] for k in ("kernel", "stride", "pad", "pads", "pad_type", "count_type",
                                                        "ceil_model", "is_global")})
    assert bits_equal(yd.cpu().numpy(), ref)


# ---------------------------------------------------------------------------------------------------------------------
# fp32 ReLU: bit-exact vs numpy (NaN only where x * slope is NaN, i.e. -inf * 0)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("slope", [0.0, 0.1, -0.5])
@pytest.mark.parametrize("count", [1, 2, 3, 5, 4 * 1025 + 3])
def test_relu_f32(backend, count, slope):
    rng = np.random.default_rng(count)
    x = rng.uniform(-3, 3, count).astype(np.float32)
    specials = np.array([-0.0, np.inf, -np.inf, 0.0, -1e-40], np.float32)
    x[:min(count, 5)] = specials[:min(count, 5)]
    x[-min(count, 5):] = specials[::-1][:min(count, 5)]
    xd, yd = f32_dev(x), nan_dev((count + 4,))
    assert lib().mnnb200_relu_f32(backend.runtime._h, C.c_void_p(xd.data_ptr()), count, C.c_float(slope),
                                  C.c_void_p(yd.data_ptr())) == 0
    backend.onSync()
    y = yd.cpu().numpy()
    assert np.isnan(y[count:]).all(), "wrote past the end"
    y = y[:count]
    with np.errstate(invalid="ignore"):
        ref = np.where(x < 0, x * np.float32(slope), x).astype(np.float32)
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(y), nan)
    assert bits_equal(y[~nan], ref[~nan])


def test_relu_f32_misaligned_is_refused(backend):
    """the kernel moves float4 words: a pointer off 16-byte alignment is an argument error, reported before any launch"""
    xd, yd = f32_dev(np.ones(64, np.float32)), nan_dev((64,))
    base_x, base_y = xd.data_ptr(), yd.data_ptr()
    rt = backend.runtime._h
    assert lib().mnnb200_relu_f32(rt, C.c_void_p(base_x + 4), 60, C.c_float(0.0), C.c_void_p(base_y)) == 5
    assert lib().mnnb200_relu_f32(rt, C.c_void_p(base_x), 60, C.c_float(0.0), C.c_void_p(base_y + 8)) == 5
    backend.onSync()
    assert np.isnan(yd.cpu().numpy()).all()


# ---------------------------------------------------------------------------------------------------------------------
# fp32 reduction over the middle axis of [outside][axis][inside]
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("inside", [1, 5, 37])
@pytest.mark.parametrize("axis", [1, 31, 32, 33, 1000])
@pytest.mark.parametrize("op", range(5), ids=["sum", "mean", "max", "min", "prod"])
def test_reduce_f32(backend, op, axis, inside):
    rng = np.random.default_rng(axis * 7 + inside + op)
    outside = 7 if inside == 1 else 3
    if op == 4:       # magnitudes near 1 keep a product of 1000 terms inside the normal range
        x = (rng.uniform(0.9, 1.1, (outside, axis, inside)) * rng.choice([-1, 1], (outside, axis, inside))).astype(np.float32)
    else:
        x = rng.uniform(-2, 2, (outside, axis, inside)).astype(np.float32)
    xd, yd = f32_dev(x), nan_dev((outside * inside,))
    assert lib().mnnb200_reduce_f32(backend.runtime._h, C.c_void_p(xd.data_ptr()), outside, axis, inside, op,
                                    C.c_void_p(yd.data_ptr())) == 0
    backend.onSync()
    y = yd.cpu().numpy().reshape(outside, inside).astype(np.float64)
    x64 = x.astype(np.float64)
    if op == 2:
        assert bits_equal(y.astype(np.float32), x.max(axis=1))
        return
    if op == 3:
        assert bits_equal(y.astype(np.float32), x.min(axis=1))
        return
    # fp32 summation of `axis` terms in any order: |err| <= (axis - 1) u sum|x| to first order; (axis + 1) 2^-23 covers it
    # with room for the second-order terms.  MEAN adds one division (relative u).  PROD: each of the axis - 1 products
    # rounds with relative error <= u, so |err| <= ((1 + u)^(axis - 1) - 1) |p| <= (axis + 1) 2^-23 |p|.
    bound_sum = (axis + 1) * 2.0 ** -23 * np.abs(x64).sum(axis=1)
    if op == 0:
        ref, tol = x64.sum(axis=1), bound_sum
    elif op == 1:
        ref = x64.mean(axis=1)
        tol = bound_sum / axis + 2 * U * np.abs(ref)
    else:
        ref = x64.prod(axis=1)
        tol = (axis + 1) * 2.0 ** -23 * np.abs(ref)
    assert (np.abs(y - ref) <= tol).all(), float((np.abs(y - ref) - tol).max())


# ---------------------------------------------------------------------------------------------------------------------
# raster (strided region copies, applied in order) and batched transpose of 4-byte elements: bit-exact vs numpy
# ---------------------------------------------------------------------------------------------------------------------
class Region(C.Structure):
    _fields_ = [("src", C.c_void_p), ("src_offset", C.c_int32), ("src_stride", C.c_int32 * 3), ("dst_offset", C.c_int32),
                ("dst_stride", C.c_int32 * 3), ("size", C.c_int32 * 3)]


def raster_numpy(dst, regions):
    for src, so, ss, do, ds, sz in regions:
        for a in range(sz[0]):
            for j in range(sz[1]):
                for k in range(sz[2]):
                    dst[do + a * ds[0] + j * ds[1] + k * ds[2]] = src[so + a * ss[0] + j * ss[1] + k * ss[2]]
    return dst


@pytest.mark.parametrize("zero_fill", [0, 1])
def test_raster_b32(backend, zero_fill):
    import torch
    rng = np.random.default_rng(11 + zero_fill)
    s0 = rng.integers(1, 2 ** 31, 600, dtype=np.int64).astype(np.int32)
    s1 = rng.integers(1, 2 ** 31, 300, dtype=np.int64).astype(np.int32)
    dst0 = np.full(500, 0x7fc0dead, np.int32)
    # (source, src_offset, src_stride, dst_offset, dst_stride, size): a 3-level transpose-like copy, a region that overlaps
    # it (written last, so it wins), a zero-size region, and a region that overwrites part of the second; elements 440-499
    # are never written
    regions = [(0, 5, (100, 1, 10), 0, (100, 10, 1), (4, 10, 10)),
               (1, 0, (0, 30, 1), 50, (0, 40, 1), (1, 5, 30)),
               (0, 0, (1, 1, 1), 0, (1, 1, 1), (3, 0, 7)),
               (0, 599, (0, 0, -7), 200, (0, 0, 3), (1, 1, 20)),
               (1, 7, (60, 3, 1), 400, (20, 5, 1), (2, 4, 5))]
    srcs = [torch.from_numpy(s0).cuda(), torch.from_numpy(s1).cuda()]
    arr = (Region * len(regions))()
    for r, (si, so, ss, do, ds, sz) in zip(arr, regions):
        r.src = srcs[si].data_ptr()
        r.src_offset, r.dst_offset = so, do
        for k in range(3):
            r.src_stride[k], r.dst_stride[k], r.size[k] = ss[k], ds[k], sz[k]
    dd = torch.from_numpy(dst0.copy()).cuda()
    assert lib().mnnb200_raster_b32(backend.runtime._h, arr, len(regions), C.c_void_p(dd.data_ptr()), dd.numel() * 4,
                                    zero_fill) == 0
    backend.onSync()
    ref = raster_numpy(np.zeros(500, np.int32) if zero_fill else dst0.copy(),
                       [([s0, s1][si], so, ss, do, ds, sz) for si, so, ss, do, ds, sz in regions])
    assert np.array_equal(dd.cpu().numpy(), ref)
    assert (ref[440:] == (0 if zero_fill else 0x7fc0dead)).all()


@pytest.mark.parametrize("batch,rows,cols", [(1, 32, 64), (2, 33, 65), (1, 1, 100), (1, 100, 1), (3, 31, 47), (4, 64, 32)])
def test_transpose_b32(backend, batch, rows, cols):
    x = np.random.default_rng(rows * cols).uniform(-1, 1, (batch, rows, cols)).astype(np.float32)
    xd, yd = f32_dev(x), nan_dev((batch * rows * cols + 8,))
    assert lib().mnnb200_transpose_b32(backend.runtime._h, C.c_void_p(xd.data_ptr()), batch, rows, cols,
                                       C.c_void_p(yd.data_ptr())) == 0
    backend.onSync()
    y = yd.cpu().numpy()
    assert np.isnan(y[batch * rows * cols:]).all(), "wrote past the end"
    assert bits_equal(y[:batch * rows * cols].reshape(batch, cols, rows), x.transpose(0, 2, 1))
