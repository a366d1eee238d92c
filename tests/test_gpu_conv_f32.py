"""fp32 convolution and its fp32 neighbours through the C ABI (-m gpu), against float64 torch on the CPU.

The split-TF32 conv (a_hi*w_hi + a_hi*w_lo + a_lo*w_hi, fp32 accumulate) must come within 1e-4 of the float64 result
(max|y - ref| / max|ref|); the depthwise conv, add and scale within 1e-5, softmax within 1e-4.  Every output is poisoned with
NaN before the run.  Two layers also report what plain TF32 (inputs and weights rounded to a 10-bit mantissa) would give."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

# (ic, oc, k, stride, pad, dilation, input h = w, batch, act)   act: 0 none, 1 ReLU, 2 ReLU6
CONV_CASES = [
    (32, 96, 1, 1, 0, 1, 56, 1, 2),        # 1x1 expand
    (24, 144, 1, 1, 0, 1, 56, 32, 2),      # 1x1, batch 32
    (64, 128, 1, 2, 0, 1, 14, 2, 0),       # 1x1 stride 2 (ResNet projection shortcut)
    (64, 64, 3, 1, 1, 1, 14, 4, 1),        # 3x3 stride 1
    (32, 64, 3, 2, 1, 1, 56, 2, 1),        # 3x3 stride 2
    (512, 512, 3, 1, 1, 1, 7, 2, 1),       # 3x3 on a 7x7 map (row stride 28 B: not TMA-describable)
    (48, 40, 3, 1, 2, 2, 14, 2, 0),        # 3x3 dilation 2, oc not a multiple of 16
    (3, 64, 7, 2, 3, 1, 112, 1, 1),        # 7x7 stride 2 stem, ic = 3
    (3, 32, 3, 2, 1, 1, 112, 1, 2),        # 3x3 stride 2 stem, ic = 3
    (160, 960, 1, 1, 0, 1, 7, 32, 2),      # 7x7 map, batch 32
    (1280, 1001, 1, 1, 0, 1, 1, 32, 0),    # classifier as a 1x1 conv: oc = 1001
]
TF32_REPORT = {1, 5}


def lib():
    from mnn_b200 import _capi
    return _capi.lib()


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def nan_dev(shape):
    import torch
    return torch.full(shape, float("nan"), dtype=torch.float32, device="cuda")


def ptr(t):
    return C.c_void_p(t.data_ptr())


def rel_err(y, ref):
    return float(np.abs(np.asarray(y, np.float64) - ref).max() / max(np.abs(ref).max(), 1e-30))


def act(y, a):
    if a >= 1:
        y = y.clamp(min=0)
    if a == 2:
        y = y.clamp(max=6)
    return y


def tf32(a):
    """round fp32 to TF32 (10-bit mantissa, nearest, ties away): what a plain TF32 tensor-core product consumes"""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def conv_ref(x, w, b, stride, pad, dil, a, groups=1):
    import torch
    y = torch.nn.functional.conv2d(torch.from_numpy(np.asarray(x, np.float64)), torch.from_numpy(np.asarray(w, np.float64)),
                                   torch.from_numpy(np.asarray(b, np.float64)), stride=stride, padding=pad, dilation=dil,
                                   groups=groups)
    return act(y, a).numpy()


def conv_inputs(rng, ic, oc, k, hw, n, depthwise=False):
    x = rng.standard_normal((n, ic, hw, hw)).astype(np.float32)
    ks = (1 if depthwise else ic) * k * k
    w = (rng.uniform(-1, 1, (oc, 1 if depthwise else ic, k, k)) * 1.2 / np.sqrt(ks)).astype(np.float32)
    b = rng.uniform(-0.5, 0.5, oc).astype(np.float32)
    return x, w, b


def desc(ic, oc, k, s, p, d, group, relu):
    from mnn_b200._capi import ConvDesc
    return ConvDesc(ic, oc, k, k, s, s, p, p, d, d, group, relu)


def create_conv(backend, ic, oc, k, s, p, d, a, w, b, depthwise=False):
    h = C.c_void_p()
    f = lib().mnnb200_dwconv_f32_create if depthwise else lib().mnnb200_conv_f32_create
    dd = desc(ic, oc, k, s, p, d, ic if depthwise else 1, int(a >= 1))
    st = f(backend.runtime._h, C.byref(dd), w.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), int(a == 2), C.byref(h))
    assert st == 0, lib().mnnb200_last_error()
    return h


def resize(h, n, hw, depthwise=False):
    oh, ow = C.c_int(0), C.c_int(0)
    f = lib().mnnb200_dwconv_f32_resize if depthwise else lib().mnnb200_conv_f32_resize
    assert f(h, n, hw, hw, C.byref(oh), C.byref(ow)) == 0, lib().mnnb200_last_error()
    return oh.value, ow.value


@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: "ic%d_oc%d_k%d_s%d_p%d_d%d_hw%d_n%d_a%d" % c)
def test_conv_f32_matches_float64(backend, case):
    ic, oc, k, s, p, d, hw, n, a = case
    rng = np.random.default_rng(ic * 131 + oc + k)
    x, w, b = conv_inputs(rng, ic, oc, k, hw, n)
    h = create_conv(backend, ic, oc, k, s, p, d, a, w, b)
    try:
        oh, ow = resize(h, n, hw)
        ref = conv_ref(x, w, b, s, p, d, a)
        assert ref.shape == (n, oc, oh, ow)
        xd, yd = dev(x), nan_dev((n, oc, oh, ow))
        assert lib().mnnb200_conv_f32_execute(h, ptr(xd), ptr(yd)) == 0, lib().mnnb200_last_error()
        backend.onSync()
        y = yd.cpu().numpy()
        assert np.isfinite(y).all()
        err = rel_err(y, ref)
        msg = f"split-TF32 rel err {err:.2e}"
        if CONV_CASES.index(case) in TF32_REPORT:
            msg += f", plain TF32 would give {rel_err(conv_ref(tf32(x), tf32(w), b, s, p, d, a), ref):.2e}"
        print(msg)
        assert err <= 1e-4, msg
        bm, macs = C.c_double(), C.c_double()
        assert lib().mnnb200_exec_cost(h, C.byref(bm), C.byref(macs)) == 0
        assert macs.value == n * oh * ow * oc * ic * k * k
    finally:
        lib().mnnb200_exec_destroy(h)


def test_conv_f32_set_pad_and_output_size(backend):
    """begin pads set after create (TF-SAME: pad 0 before, 1 after) with the output size passed in, as the plugin resizes"""
    ic, oc, k, s, hw, n = 16, 24, 3, 2, 14, 2
    rng = np.random.default_rng(7)
    x, w, b = conv_inputs(rng, ic, oc, k, hw, n)
    h = create_conv(backend, ic, oc, k, s, 1, 1, 0, w, b)
    try:
        assert lib().mnnb200_conv_f32_set_pad(h, 0, 0) == 0
        oh, ow = C.c_int(7), C.c_int(7)
        assert lib().mnnb200_conv_f32_resize(h, n, hw, hw, C.byref(oh), C.byref(ow)) == 0
        xpad = np.pad(x, ((0, 0), (0, 0), (0, 1), (0, 1)))
        ref = conv_ref(xpad, w, b, s, 0, 1, 0)
        assert ref.shape == (n, oc, 7, 7)
        xd, yd = dev(x), nan_dev((n, oc, 7, 7))
        assert lib().mnnb200_conv_f32_execute(h, ptr(xd), ptr(yd)) == 0
        backend.onSync()
        assert rel_err(yd.cpu().numpy(), ref) <= 1e-4
    finally:
        lib().mnnb200_exec_destroy(h)


def test_conv_f32_declines_grouped(backend):
    w = np.zeros((8, 4, 3, 3), np.float32)
    h = C.c_void_p()
    dd = desc(8, 8, 3, 1, 1, 1, 2, 0)
    assert lib().mnnb200_conv_f32_create(backend.runtime._h, C.byref(dd), w.ctypes.data_as(C.c_void_p), None, 0, C.byref(h)) == 2
    assert not h.value


@pytest.mark.parametrize("case", [(32, 3, 1, 1, 1, 112, 1, 2), (144, 3, 2, 1, 1, 56, 2, 2), (960, 3, 1, 1, 1, 7, 32, 1),
                                  (64, 5, 1, 4, 2, 14, 2, 0), (24, 3, 2, 0, 1, 15, 3, 1)],
                         ids=lambda c: "c%d_k%d_s%d_p%d_d%d_hw%d_n%d_a%d" % c)
def test_dwconv_f32_matches_float64(backend, case):
    c, k, s, p, d, hw, n, a = case
    rng = np.random.default_rng(c + k * 7 + hw)
    x, w, b = conv_inputs(rng, c, c, k, hw, n, depthwise=True)
    h = create_conv(backend, c, c, k, s, p, d, a, w, b, depthwise=True)
    try:
        oh, ow = resize(h, n, hw, depthwise=True)
        ref = conv_ref(x, w, b, s, p, d, a, groups=c)
        assert ref.shape == (n, c, oh, ow)
        xd, yd = dev(x), nan_dev((n, c, oh, ow))
        assert lib().mnnb200_dwconv_f32_execute(h, ptr(xd), ptr(yd)) == 0, lib().mnnb200_last_error()
        backend.onSync()
        assert rel_err(yd.cpu().numpy(), ref) <= 1e-5
    finally:
        lib().mnnb200_exec_destroy(h)


@pytest.mark.parametrize("count", [1, 7, 4096, 32 * 24 * 56 * 56 + 3])
def test_binary_add_f32(backend, count):
    rng = np.random.default_rng(count)
    a, b = rng.standard_normal(count).astype(np.float32), rng.standard_normal(count).astype(np.float32)
    ad, bd, yd = dev(a), dev(b), nan_dev((count,))
    assert lib().mnnb200_binary_add_f32(backend.runtime._h, ptr(ad), ptr(bd), ptr(yd), count) == 0
    backend.onSync()
    ref = a.astype(np.float64) + b
    assert rel_err(yd.cpu().numpy(), ref) <= 1e-5
    # an unaligned view takes the scalar path
    if count > 8:
        yd2 = nan_dev((count,))
        assert lib().mnnb200_binary_add_f32(backend.runtime._h, C.c_void_p(ad.data_ptr() + 4), ptr(bd), ptr(yd2), count - 1) == 0
        backend.onSync()
        assert rel_err(yd2.cpu().numpy()[:-1], a[1:].astype(np.float64) + b[:-1]) <= 1e-5


@pytest.mark.parametrize("shape", [(2, 64, 56, 56), (32, 2048, 7, 7), (1, 3, 5, 1)])
def test_scale_f32(backend, shape):
    n, c, hh, ww = shape
    rng = np.random.default_rng(c)
    x = rng.standard_normal(shape).astype(np.float32)
    s, b = rng.uniform(0.5, 1.5, c).astype(np.float32), rng.uniform(-0.2, 0.2, c).astype(np.float32)
    h = C.c_void_p()
    assert lib().mnnb200_scale_f32_create(backend.runtime._h, c, s.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p),
                                          C.byref(h)) == 0
    try:
        assert lib().mnnb200_scale_f32_resize(h, n, hh, ww) == 0
        xd, yd = dev(x), nan_dev(shape)
        assert lib().mnnb200_scale_f32_execute(h, ptr(xd), ptr(yd)) == 0
        backend.onSync()
        ref = x.astype(np.float64) * s[None, :, None, None] + b[None, :, None, None]
        assert rel_err(yd.cpu().numpy(), ref) <= 1e-5
    finally:
        lib().mnnb200_exec_destroy(h)


@pytest.mark.parametrize("view", [(32, 1001, 1), (4, 10, 49), (3, 70, 5), (1, 1, 1)])
def test_softmax_f32(backend, view):
    import torch
    outside, axis, inside = view
    rng = np.random.default_rng(axis)
    x = (rng.standard_normal(view) * 4).astype(np.float32)
    xd, yd = dev(x), nan_dev(view)
    assert lib().mnnb200_softmax_f32(backend.runtime._h, ptr(xd), outside, axis, inside, ptr(yd)) == 0
    backend.onSync()
    ref = torch.softmax(torch.from_numpy(x.astype(np.float64)), dim=1).numpy()
    assert rel_err(yd.cpu().numpy(), ref) <= 1e-4


def test_float_stack_repeatable_and_graph_replay(backend):
    """conv -> depthwise -> conv -> add -> scale -> softmax: two eager runs give equal bits, and so does a replay of the same
    sequence captured as one CUDA graph on the runtime's stream"""
    import torch
    rng = np.random.default_rng(3)
    n, c, hw = 4, 32, 28
    x = rng.standard_normal((n, c, hw, hw)).astype(np.float32)
    _, w1, b1 = conv_inputs(rng, c, 96, 1, hw, n)
    _, wd, bd = conv_inputs(rng, 96, 96, 3, hw, n, depthwise=True)
    _, w2, b2 = conv_inputs(rng, 96, c, 1, hw, n)
    s, sb = rng.uniform(0.5, 1.5, c).astype(np.float32), rng.uniform(-0.2, 0.2, c).astype(np.float32)
    h1 = create_conv(backend, c, 96, 1, 1, 0, 1, 2, w1, b1)
    hd = create_conv(backend, 96, 96, 3, 1, 1, 1, 2, wd, bd, depthwise=True)
    h2 = create_conv(backend, 96, c, 1, 1, 0, 1, 0, w2, b2)
    hs = C.c_void_p()
    assert lib().mnnb200_scale_f32_create(backend.runtime._h, c, s.ctypes.data_as(C.c_void_p), sb.ctypes.data_as(C.c_void_p),
                                          C.byref(hs)) == 0
    g = C.c_void_p()
    try:
        resize(h1, n, hw)
        resize(hd, n, hw, depthwise=True)
        resize(h2, n, hw)
        assert lib().mnnb200_scale_f32_resize(hs, n, hw, hw) == 0
        xd = dev(x)
        t1, t2, t3, t4, t5 = (torch.empty((n, ch, hw, hw), device="cuda") for ch in (96, 96, c, c, c))
        out = torch.empty((n, c, hw, hw), device="cuda")
        rt = backend.runtime._h

        def forward():
            assert lib().mnnb200_conv_f32_execute(h1, ptr(xd), ptr(t1)) == 0
            assert lib().mnnb200_dwconv_f32_execute(hd, ptr(t1), ptr(t2)) == 0
            assert lib().mnnb200_conv_f32_execute(h2, ptr(t2), ptr(t3)) == 0
            assert lib().mnnb200_binary_add_f32(rt, ptr(t3), ptr(xd), ptr(t4), t4.numel()) == 0
            assert lib().mnnb200_scale_f32_execute(hs, ptr(t4), ptr(t5)) == 0
            assert lib().mnnb200_softmax_f32(rt, ptr(t5), n, c, hw * hw, ptr(out)) == 0

        forward()
        backend.onSync()
        first = out.cpu().numpy()
        mid = t4.cpu().numpy()
        out.fill_(float("nan"))
        forward()
        backend.onSync()
        assert np.array_equal(out.cpu().numpy(), first)
        out.fill_(float("nan"))
        backend.onSync()
        assert lib().mnnb200_graph_begin_capture(rt) == 0
        forward()
        assert lib().mnnb200_graph_end_capture(rt, C.byref(g)) == 0, lib().mnnb200_last_error()
        assert lib().mnnb200_graph_launch(rt, g) == 0
        backend.onSync()
        assert np.array_equal(out.cpu().numpy(), first)
        # and the chain itself against float64
        r1 = conv_ref(x, w1, b1, 1, 0, 1, 2)
        r2 = conv_ref(r1, wd, bd, 1, 1, 1, 2, groups=96)
        r4 = conv_ref(r2, w2, b2, 1, 0, 1, 0) + x
        assert rel_err(mid, r4) <= 1e-4
        r5 = r4 * s[None, :, None, None] + sb[None, :, None, None]
        ref = torch.softmax(torch.from_numpy(r5), dim=1).numpy()
        assert rel_err(first, ref) <= 1e-4
    finally:
        if g.value:
            lib().mnnb200_graph_destroy(g)
        for h in (h1, hd, h2, hs):
            lib().mnnb200_exec_destroy(h)


@pytest.mark.parametrize("op_type", ["Convolution", "ConvolutionDepthwise"])
def test_float_conv_through_backend_mirror(backend, op_type):
    """Backend.onCreate -> onResize (output shape) -> onExecute for the float conv creators of the Python mirror"""
    from mnn_b200.backend import Op, Tensor
    dw = op_type == "ConvolutionDepthwise"
    n, ic, oc, hw = 2, 24, 24 if dw else 40, 15
    rng = np.random.default_rng(11)
    x, w, b = conv_inputs(rng, ic, oc, 3, hw, n, depthwise=dw)
    op = Op(type=op_type, conv=dict(ic=ic, oc=oc, kernel=(3, 3), stride=(2, 2), pad=(1, 1), group=ic if dw else 1, relu=True),
            weight=w, bias=b, relu6=True)
    xin = backend.onAcquire(Tensor((n, ic, hw, hw), "float"))
    backend.onCopyBuffer(x, xin)
    yout = Tensor((n, oc, 1, 1), "float")
    ex = backend.onCreate([xin], [yout], op)
    assert ex is not None and ex.onResize([xin], [yout]) == 0
    assert yout.shape == (n, oc, 8, 8)
    backend.onAcquire(yout)
    yout.data.fill_(float("nan"))
    assert ex.onExecute([xin], [yout]) == 0
    backend.onSync()
    ref = conv_ref(x, w, b, 2, 1, 1, 2, groups=ic if dw else 1)
    assert rel_err(backend.onCopyBuffer(yout, "same"), ref) <= 1e-4
    grouped = Op(type="Convolution", conv=dict(ic=ic, oc=oc, kernel=(3, 3), group=2), weight=w, bias=b)
    assert backend.onCreate([xin], [yout], grouped) is None
