"""fp32 Deconvolution through the C ABI (-m gpu), against the float64 oracle (oracle/deconv_oracle.py).

Every output of the split-TF32 transposed convolution must lie within the error model of tests/test_gpu_conv_f32.py
(conv_tolerance) with Kp the K of the output's own phase (its taps * cp8, rounded up to whole K blocks), and all of them together
within 1e-4 of max|ref|; the depthwise gather within its fmaf chain's model and 1e-5.  Inputs sit between NaN guard bands 4 bytes
past 16-byte alignment and outputs in NaN-filled buffers, so a read outside x, a write outside y or an output left unwritten
shows.  The cell matrix derives its shapes from the SM count with resize's own tile-width rule and reads the launch back through
mnnb200_deconv_f32_plan."""
import ctypes as C

import numpy as np
import pytest

from oracle.deconv_oracle import deconv_f32, natural_out, pair
from tests.golden import make_deconv_golden as G
from tests.test_deconv_cpu import golden_check
from tests.test_gpu_conv_f32 import GUARD, check_elements, conv_tolerance, dw_tolerance, guarded, ptr, rel_err, sm_count

pytestmark = pytest.mark.gpu

NOT_SUPPORT, NO_EXECUTION, INVALID_VALUE = 2, 4, 5
PLAN_FIELDS = ("bn", "n_chunks", "phases", "m_tiles", "num_kb", "stages", "taps")


def lib():
    from mnn_b200 import _capi
    return _capi.lib()


def dlib():
    from mnn_b200 import _capi
    return _capi.deconv_lib()


def inputs(rng, ic, oc, k, hw, n, depthwise=False):
    (kh, kw), (ih, iw) = pair(k), pair(hw)
    x = rng.standard_normal((n, ic, ih, iw)).astype(np.float32)
    shape = (ic, kh, kw) if depthwise else (ic, oc, kh, kw)
    w = (rng.uniform(-1, 1, shape) * 1.2 / np.sqrt((1 if depthwise else ic) * kh * kw)).astype(np.float32)
    b = rng.uniform(-0.5, 0.5, oc).astype(np.float32)
    return x, w, b


def create(backend, ic, oc, k, s, p, d, a, w, b, depthwise=False):
    from mnn_b200._capi import ConvDesc
    (kh, kw), (sh, sw), (ph, pw), (dh, dw) = pair(k), pair(s), pair(p), pair(d)
    dd = ConvDesc(ic, oc, kh, kw, sh, sw, ph, pw, dh, dw, ic if depthwise else 1, int(a >= 1))
    h = C.c_void_p()
    f = dlib().mnnb200_dwdeconv_f32_create if depthwise else dlib().mnnb200_deconv_f32_create
    st = f(backend.runtime._h, C.byref(dd), w.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), int(a == 2), C.byref(h))
    assert st == 0, lib().mnnb200_last_error()
    return h


def resize_status(h, n, hw, out=None, depthwise=False):
    (ih, iw), (oh0, ow0) = pair(hw), out or (0, 0)
    oh, ow = C.c_int(oh0), C.c_int(ow0)
    f = dlib().mnnb200_dwdeconv_f32_resize if depthwise else dlib().mnnb200_deconv_f32_resize
    return f(h, n, ih, iw, C.byref(oh), C.byref(ow)), (oh.value, ow.value)


def resize(h, n, hw, out=None, depthwise=False):
    st, ohw = resize_status(h, n, hw, out, depthwise)
    assert st == 0, lib().mnnb200_last_error()
    return ohw


def plan(h):
    f = (C.c_int * len(PLAN_FIELDS))()
    assert dlib().mnnb200_deconv_f32_plan(h, f, len(f)) == 0, lib().mnnb200_last_error()
    return dict(zip(PLAN_FIELDS, f))


def execute_with(backend, f, h, x, out_shape):
    """run f(h, x, y) with x and y guarded; the device output after checking that neither guard band was written"""
    import torch
    xb, xd = guarded(x.shape, x)
    yb, yd = guarded(out_shape)
    assert f(h, ptr(xd), ptr(yd)) == 0, lib().mnnb200_last_error()
    backend.onSync()
    for buf, t, what in ((xb, xd, "x"), (yb, yd, "y")):
        g = torch.cat([buf[:GUARD], buf[GUARD + t.numel():]])
        assert bool(torch.isnan(g).all()), f"{int((~torch.isnan(g)).sum())} floats of {what}'s guard bands were written"
    return yd


def axis_taps(r, s, d, k):
    """kernel positions of one axis in phase r: k * d = r (mod s)"""
    return [t for t in range(k) if (t * d) % s == r]


def phase_kp(ic, k, s, p, d, out_hw):
    """[oh][ow] K of each output's phase as the kernel pads it: taps * cp8 rounded up to 32"""
    (kh, kw), (sh, sw), (ph, pw), (dh, dw) = pair(k), pair(s), pair(p), pair(d)
    cp8 = -(-ic // 8) * 8
    ty = np.array([len(axis_taps((o + ph) % sh, sh, dh, kh)) for o in range(out_hw[0])])
    tx = np.array([len(axis_taps((o + pw) % sw, sw, dw, kw)) for o in range(out_hw[1])])
    return -(-(ty[:, None] * tx[None, :] * cp8) // 32) * 32


def run(backend, h, x, w, b, k, s, p, d, a, out_hw, what=""):
    """execute the resized deconvolution h on guarded x / y and check every output per element against float64 within its
    phase's bound and by the max-norm contract: (rel err, plan, ref, S, y)"""
    pl = plan(h)
    n, ic = x.shape[:2]
    oc = w.shape[1]
    y = execute_with(backend, dlib().mnnb200_deconv_f32_execute, h, x, (n, oc) + tuple(out_hw)).cpu().numpy()
    ref, S = deconv_f32(x, w, b, s, p, d, a, out_hw=tuple(out_hw))
    tol = conv_tolerance(S, b, phase_kp(ic, k, s, p, d, out_hw)[None, None])
    check_elements(y, ref, tol, what)
    err = rel_err(y, ref)
    assert err <= 1e-4, f"{what}: split-TF32 rel err {err:.2e}"
    return err, pl, ref, S, y


def expected_taps(k, s, d):
    (kh, kw), (sh, sw), (dh, dw) = pair(k), pair(s), pair(d)
    return max(len(axis_taps(ry, sh, dh, kh)) * len(axis_taps(rx, sw, dw, kw)) for ry in range(sh) for rx in range(sw))


# name: ic, oc, kernel, stride, pad, dilation, (ih, iw), batch, act, explicit output (None: natural)
CASES = {
    "k4_s2_p1_simplebaseline": (64, 40, 4, 2, 1, 1, (8, 6), 2, 1, None),
    "k2_s2_unet": (48, 24, 2, 2, 0, 1, 14, 2, 0, None),
    "k3_s2_p1_outpad1": (13, 20, 3, 2, 1, 1, 9, 2, 2, (18, 18)),
    "k16_s8_p4_fcn": (21, 21, 16, 8, 4, 1, 7, 1, 0, None),
    "k3_s2_d2": (8, 16, 3, 2, 1, 2, 10, 2, 0, None),
    "k1_s2_no_taps": (5, 24, 1, 2, 0, 1, 9, 2, 1, None),
    "k2_s3_no_taps": (16, 24, 2, 3, 0, 1, 8, 2, 0, None),
    "k3_s2_p4_beyond": (5, 24, 3, 2, 4, 1, 12, 2, 0, None),
    "k3x5_s2x3_d1x2_p1x2_ic1": (1, 33, (3, 5), (2, 3), (1, 2), (1, 2), (11, 7), 2, 1, None),
    "k5x3_s3x2_p2x0_ic13": (13, 36, (5, 3), (3, 2), (2, 0), 1, (9, 12), 2, 0, None),
    "k3_s1_p1_ic5": (5, 20, 3, 1, 1, 1, (13, 11), 2, 2, None),
    "k4_s4_outpads_unreached": (13, 24, 3, 4, 0, 1, (5, 6), 2, 0, (20, 23)),
    "k3_s2_same": (16, 40, 3, 2, 0, 1, (7, 9), 2, 0, (14, 18)),
}


@pytest.mark.parametrize("name", list(CASES))
def test_deconv_f32_matches_float64(backend, name):
    ic, oc, k, s, p, d, hw, n, a, out = CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    x, w, b = inputs(rng, ic, oc, k, hw, n)
    h = create(backend, ic, oc, k, s, p, d, a, w, b)
    try:
        ohw = resize(h, n, hw, out)
        (kh, kw), (sh, sw), (ph, pw), (dh, dw) = pair(k), pair(s), pair(p), pair(d)
        assert ohw == (out or (natural_out(pair(hw)[0], kh, sh, ph, dh), natural_out(pair(hw)[1], kw, sw, pw, dw)))
        err, pl, ref, S, _ = run(backend, h, x, w, b, k, s, p, d, a, ohw, what=name)
        assert (pl["phases"], pl["taps"]) == (sh * sw, expected_taps(k, s, d))
        print(f"{name}: {n} x {hw} -> {ohw}, plan {pl}, rel err {err:.2e}")
        if "no_taps" in name or "unreached" in name:
            bias_only = (S == 0).all(axis=(0, 1))
            assert bias_only.any(), "wanted outputs that no tap reaches"
            want = np.broadcast_to(np.maximum(b.astype(np.float64), 0) if a else b.astype(np.float64),
                                   (n, bias_only.sum(), oc)).transpose(0, 2, 1)
            assert np.array_equal(ref[:, :, bias_only], want)
        bm, macs = C.c_double(), C.c_double()
        assert lib().mnnb200_exec_cost(h, C.byref(bm), C.byref(macs)) == 0
        assert macs.value == n * pair(hw)[0] * pair(hw)[1] * ic * oc * kh * kw
    finally:
        lib().mnnb200_exec_destroy(h)


def plan_bn(oc, m_tiles, sms):
    """mnnb200_deconv_f32_resize: the widest tile oc wants, halved while the work items (all phases) would not fill the SMs"""
    bn = 32 if oc <= 32 else 64 if oc <= 64 else 128
    while bn > 32 and m_tiles * -(-oc // bn) < sms:
        bn //= 2
    return bn


# name: (ic, kernel, pad, act).  kb1: 2x2 stride 2, one tap per phase, ic 20 (cp8 24): one K block.  ring: 4x4 stride 2, four taps
# per phase, ic 80: K = 320 = 10 blocks, more than any width's ring holds and not a multiple of it
CELLS = {"kb1": (20, 2, 0, 2), "ring": (80, 4, 1, 1)}


@pytest.mark.parametrize("bn", [32, 64, 128])
@pytest.mark.parametrize("cell", list(CELLS))
def test_deconv_f32_cell_matrix(backend, bn, cell):
    """each tile width with one K block and with a wrapping ring: more items than SMs, so a CTA's items fall in different phases
    and (chunks not dividing the SM count) different n chunks, a ragged last n chunk, ragged last M tiles of every phase and an M
    tile across two images"""
    sms = sm_count()
    ic, k, p, a = CELLS[cell]
    chunks = next(c for c in range(2, 64) if sms % c)
    oc = bn * (chunks - 1) + bn // 2 + 3 if bn > 32 else 27
    n, iw = 2, 13
    ih = next(ih for ih in range(2, 400) if (n * ih * iw) % 128 and (ih * iw) % 128 and
              4 * -(-n * ih * iw // 128) * -(-oc // bn) > sms and plan_bn(oc, 4 * -(-n * ih * iw // 128), sms) == bn)
    rng = np.random.default_rng(bn * 10 + k)
    x, w, b = inputs(rng, ic, oc, k, (ih, iw), n)
    h = create(backend, ic, oc, k, 2, p, 1, a, w, b)
    try:
        ohw = resize(h, n, (ih, iw))
        assert ohw == (2 * ih, 2 * iw)
        err, pl, _, _, _ = run(backend, h, x, w, b, k, 2, p, 1, a, ohw, what=f"bn {bn} {cell}")
        m_phase = -(-n * ih * iw // 128)
        items = 4 * m_phase * pl["n_chunks"]
        print(f"BN {bn} {cell}: plan {pl}, oc {oc}, {n} x {ih}x{iw}, {items} items on {sms} SMs, rel err {err:.2e}")
        assert (pl["bn"], pl["m_tiles"], pl["n_chunks"], pl["phases"]) == (bn, m_phase, -(-oc // bn), 4)
        if cell == "kb1":
            assert pl["num_kb"] == 1
        else:
            assert pl["num_kb"] == 10 and pl["num_kb"] > pl["stages"] and pl["num_kb"] % pl["stages"], pl
        assert items > sms and m_phase * pl["n_chunks"] < sms, "a CTA's items must span phases"
        assert oc % bn, "ragged last n chunk"
    finally:
        lib().mnnb200_exec_destroy(h)


def test_deconv_f32_re_resize_matches_fresh_plan(backend):
    """one execution resized batch 1 (bn 32) -> a shape that plans bn 128 -> new pads -> batch 1 again: each plan equals the
    plan of a fresh execution resized once to that shape, and every output is checked"""
    sms = sm_count()
    ic, oc, k, s, a = 24, 200, 4, 2, 1
    rng = np.random.default_rng(200)
    _, w, b = inputs(rng, ic, oc, k, 1, 1)
    h = create(backend, ic, oc, k, s, 1, 1, a, w, b)
    ih128 = next(i for i in range(2, 400) if plan_bn(oc, 4 * -(-2 * i * 13 // 128), sms) == 128)
    try:
        widths = []
        for n, hw, pad in ((1, (5, 7), (1, 1)), (2, (ih128, 13), (1, 1)), (1, (6, 5), (0, 2))):
            if pad != (1, 1):
                assert dlib().mnnb200_deconv_f32_set_pad(h, *pad) == 0
            x = rng.standard_normal((n, ic) + hw).astype(np.float32)
            ohw = resize(h, n, hw)
            err, pl, _, _, _ = run(backend, h, x, w, b, k, s, pad, 1, a, ohw, what=f"resize to {n} x {hw}")
            fresh = create(backend, ic, oc, k, s, pad, 1, a, w, b)
            try:
                resize(fresh, n, hw)
                assert plan(fresh) == pl
            finally:
                lib().mnnb200_exec_destroy(fresh)
            widths.append(pl["bn"])
        assert widths == [32, 128, 32]
    finally:
        lib().mnnb200_exec_destroy(h)


def test_deconv_f32_set_pad_and_output_shape(backend):
    """TF-SAME (ConvolutionCommon::convolutionTransposePad: pad = ((ih - 1) * s + k - oh) / 2 before) with the output size
    passed in, as the plugin resizes"""
    ic, oc, k, s, n, (ih, iw) = 12, 20, 5, 2, 2, (7, 10)
    rng = np.random.default_rng(9)
    x, w, b = inputs(rng, ic, oc, k, (ih, iw), n)
    h = create(backend, ic, oc, k, s, 0, 1, 0, w, b)
    try:
        out = (ih * s, iw * s)
        pad = (((ih - 1) * s + k - out[0]) // 2, ((iw - 1) * s + k - out[1]) // 2)
        assert dlib().mnnb200_deconv_f32_set_pad(h, *pad) == 0
        assert resize(h, n, (ih, iw), out=out) == out
        run(backend, h, x, w, b, k, s, pad, 1, 0, out, what="SAME")
    finally:
        lib().mnnb200_exec_destroy(h)


def test_deconv_f32_plan_query(backend):
    rng = np.random.default_rng(5)
    _, w, b = inputs(rng, 8, 8, 3, 1, 1)
    _, wd, bd = inputs(rng, 8, 8, 3, 1, 1, depthwise=True)
    h = create(backend, 8, 8, 3, 2, 1, 1, 0, w, b)
    hd = create(backend, 8, 8, 3, 2, 1, 1, 0, wd, bd, depthwise=True)
    try:
        f = (C.c_int * 7)(*([-7] * 7))
        assert dlib().mnnb200_deconv_f32_plan(h, f, 7) == NO_EXECUTION
        assert dlib().mnnb200_deconv_f32_plan(hd, f, 7) == INVALID_VALUE
        assert dlib().mnnb200_deconv_f32_plan(None, f, 7) == INVALID_VALUE
        resize(h, 1, 5)
        resize(hd, 1, 5, depthwise=True)
        assert dlib().mnnb200_deconv_f32_plan(h, None, 7) == INVALID_VALUE
        assert list(f) == [-7] * 7
        assert dlib().mnnb200_deconv_f32_plan(h, f, 3) == 0
        assert list(f) == [32, 1, 4, -7, -7, -7, -7]
        pl = plan(h)
        assert plan(h) == pl == dict(bn=32, n_chunks=1, phases=4, m_tiles=1, num_kb=1, stages=pl["stages"], taps=4)
        assert pl["stages"] > 0
    finally:
        lib().mnnb200_exec_destroy(h)
        lib().mnnb200_exec_destroy(hd)


def test_deconv_f32_refusals_keep_the_plan(backend):
    """NOT_SUPPORT one past each 32-bit limit (n*oh*ow <= 2^31 - 129, n*ic*ih*iw and n*oc*oh*ow <= 2^31 - 1), for an empty
    tensor and for an output past what pads and strides produce, each accepting the limit itself; a refused resize leaves the
    plan as it was.  Host arithmetic only: nothing is launched."""
    rng = np.random.default_rng(6)
    _, w1, b1 = inputs(rng, 1, 1, 1, 1, 1)
    _, w2, b2 = inputs(rng, 1, 1024, 1, 1, 1)
    _, w3, b3 = inputs(rng, 4, 4, 3, 1, 1)
    h1 = create(backend, 1, 1, 1, 1, 0, 1, 0, w1, b1)
    h2 = create(backend, 1, 1024, 1, 1, 0, 1, 0, w2, b2)
    h3 = create(backend, 4, 4, 3, 2, 1, 1, 0, w3, b3)
    lim = 2 ** 31 - 1
    try:
        def refused(h, n, hw, out):
            before = plan(h)
            st, _ = resize_status(h, n, hw, out)
            assert st == NOT_SUPPORT, (n, hw, out)
            assert plan(h) == before

        # 1x1 stride 1: the output may be the input's size at most
        assert resize_status(h1, 1, (lim - 128, 1), (lim - 128, 1))[0] == 0
        refused(h1, 1, ((lim - 127) // 128, 128), ((lim - 127) // 128, 128))
        assert resize_status(h1, 1, (lim, 1), (1, 1))[0] == 0
        refused(h1, 2, (2 ** 30, 1), (1, 1))
        assert resize_status(h2, 1, (2 ** 21 - 1, 1), (2 ** 21 - 1, 1))[0] == 0
        refused(h2, 1, (2048, 1024), (2048, 1024))
        # 3x3 stride 2 begin pad 1 from 5x5: natural 9; no end pad and an out-pad of stride - 1 reach 11, 12 is past
        assert resize(h3, 1, 5) == (9, 9)
        assert resize(h3, 1, 5, out=(11, 11)) == (11, 11)
        refused(h3, 1, 5, (12, 11))
        refused(h3, 1, 5, (11, 12))
        refused(h3, 0, 5, None)
        refused(h3, 1, (0, 5), None)
    finally:
        for h in (h1, h2, h3):
            lib().mnnb200_exec_destroy(h)


def test_deconv_f32_declines_grouped_and_wide_strides(backend):
    from mnn_b200._capi import ConvDesc
    w = np.zeros((8, 4, 3, 3), np.float32)
    for dd in (ConvDesc(8, 8, 3, 3, 1, 1, 1, 1, 1, 1, 2, 0), ConvDesc(8, 4, 3, 3, 17, 1, 0, 0, 1, 1, 1, 0)):
        h = C.c_void_p()
        assert dlib().mnnb200_deconv_f32_create(backend.runtime._h, C.byref(dd), w.ctypes.data_as(C.c_void_p), None, 0,
                                               C.byref(h)) == NOT_SUPPORT
        assert not h.value
    dd = ConvDesc(8, 8, 3, 3, 1, 1, 1, 1, 1, 1, 4, 0)
    h = C.c_void_p()
    assert dlib().mnnb200_dwdeconv_f32_create(backend.runtime._h, C.byref(dd), w.ctypes.data_as(C.c_void_p), None, 0,
                                             C.byref(h)) == NOT_SUPPORT


# name: channels, kernel, stride, pad, dilation, (ih, iw), batch, act, explicit output
DW_CASES = {
    "c32_k4_s2_p1": (32, 4, 2, 1, 1, (14, 10), 2, 1, None),
    "c24_k3_s2_p1_outpad": (24, 3, 2, 1, 1, (9, 7), 2, 2, (18, 14)),
    "c7_k3x5_s1x3_p0x2_d2x1": (7, (3, 5), (1, 3), (0, 2), (2, 1), (8, 6), 3, 0, None),
    "c16_k1_s2_no_taps": (16, 1, 2, 0, 1, (6, 5), 2, 0, None),
}


@pytest.mark.parametrize("name", list(DW_CASES))
def test_dwdeconv_f32_matches_float64(backend, name):
    c, k, s, p, d, hw, n, a, out = DW_CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    x, w, b = inputs(rng, c, c, k, hw, n, depthwise=True)
    h = create(backend, c, c, k, s, p, d, a, w, b, depthwise=True)
    try:
        ohw = resize(h, n, hw, out, depthwise=True)
        y = execute_with(backend, dlib().mnnb200_dwdeconv_f32_execute, h, x, (n, c) + ohw).cpu().numpy()
        ref, S = deconv_f32(x, w, b, s, p, d, a, out_hw=ohw, depthwise=True)
        check_elements(y, ref, dw_tolerance(S, b, max(1, int(np.prod(pair(k))))), name)
        assert rel_err(y, ref) <= 1e-5
    finally:
        lib().mnnb200_exec_destroy(h)


def test_deconv_between_convs_graph_replay(backend):
    """conv -> deconv -> depthwise deconv -> conv through the C ABI: two eager runs give equal bits, and so does a replay of the
    sequence captured as one CUDA graph, after the input is rewritten in place (the replay reads the new input)"""
    import torch
    from tests.test_gpu_conv_f32 import conv_inputs, conv_ref, create_conv, resize as conv_resize
    rng = np.random.default_rng(3)
    n, c, hw = 2, 16, 12
    x1 = rng.standard_normal((n, c, hw, hw)).astype(np.float32)
    x2 = rng.standard_normal((n, c, hw, hw)).astype(np.float32)
    _, w1, b1 = conv_inputs(rng, c, 32, 3, hw, n)
    _, wd, bd = inputs(rng, 32, 24, 4, 1, 1)
    _, wdd, bdd = inputs(rng, 24, 24, 3, 1, 1, depthwise=True)
    _, w2, b2 = conv_inputs(rng, 24, 8, 1, hw, n)
    h1 = create_conv(backend, c, 32, 3, 1, 1, 1, 1, w1, b1)
    hd = create(backend, 32, 24, 4, 2, 1, 1, 1, wd, bd)
    hdd = create(backend, 24, 24, 3, 1, 1, 1, 0, wdd, bdd, depthwise=True)
    h2 = create_conv(backend, 24, 8, 1, 1, 0, 1, 0, w2, b2)
    g = C.c_void_p()
    try:
        conv_resize(h1, n, hw)
        assert resize(hd, n, hw) == (2 * hw, 2 * hw)
        assert resize(hdd, n, 2 * hw, depthwise=True) == (2 * hw, 2 * hw)
        conv_resize(h2, n, 2 * hw)
        xd = torch.from_numpy(x1).cuda()
        t1 = torch.empty((n, 32, hw, hw), device="cuda")
        t2, t3 = (torch.empty((n, 24, 2 * hw, 2 * hw), device="cuda") for _ in range(2))
        out = torch.empty((n, 8, 2 * hw, 2 * hw), device="cuda")
        rt = backend.runtime._h

        def forward():
            assert lib().mnnb200_conv_f32_execute(h1, ptr(xd), ptr(t1)) == 0
            assert dlib().mnnb200_deconv_f32_execute(hd, ptr(t1), ptr(t2)) == 0
            assert dlib().mnnb200_dwdeconv_f32_execute(hdd, ptr(t2), ptr(t3)) == 0
            assert lib().mnnb200_conv_f32_execute(h2, ptr(t3), ptr(out)) == 0

        def reference(x):
            r1 = conv_ref(x, w1, b1, 1, 1, 1, 1)
            r2, _ = deconv_f32(r1, wd, bd, 2, 1, 1, 1)
            r3, _ = deconv_f32(r2, wdd, bdd, 1, 1, 1, 0, depthwise=True)
            return conv_ref(r3, w2, b2, 1, 0, 1, 0)

        forward()
        backend.onSync()
        first = out.cpu().numpy()
        assert rel_err(first, reference(x1)) <= 1e-4
        out.fill_(float("nan"))
        forward()
        backend.onSync()
        assert np.array_equal(out.cpu().numpy(), first)
        assert lib().mnnb200_graph_begin_capture(rt) == 0
        forward()
        assert lib().mnnb200_graph_end_capture(rt, C.byref(g)) == 0, lib().mnnb200_last_error()
        xd.copy_(torch.from_numpy(x2))
        out.fill_(float("nan"))
        backend.onSync()
        assert lib().mnnb200_graph_launch(rt, g) == 0
        backend.onSync()
        second = out.cpu().numpy()
        assert rel_err(second, reference(x2)) <= 1e-4
        forward()
        backend.onSync()
        assert np.array_equal(out.cpu().numpy(), second)
    finally:
        if g.value:
            lib().mnnb200_graph_destroy(g)
        for h in (h1, hd, hdd, h2):
            lib().mnnb200_exec_destroy(h)


@pytest.mark.parametrize("op_type", ["DeconvF32", "DwDeconvF32"])
def test_deconv_through_backend_mirror(backend, op_type):
    """Backend.onCreate -> onResize (output shape) -> onExecute for the deconvolution creators of the Python mirror"""
    from mnn_b200.backend import Op, Tensor
    dw = op_type == "DwDeconvF32"
    n, ic, oc, hw = 2, 24, 24 if dw else 40, 9
    rng = np.random.default_rng(11)
    x, w, b = inputs(rng, ic, oc, 4, hw, n, depthwise=dw)
    op = Op(type=op_type, conv=dict(ic=ic, oc=oc, kernel=(4, 4), stride=(2, 2), pad=(1, 1), group=ic if dw else 1, relu=True),
            weight=w, bias=b, relu6=True)
    xin = backend.onAcquire(Tensor((n, ic, hw, hw), "float"))
    backend.onCopyBuffer(x, xin)
    yout = Tensor((n, oc, 1, 1), "float")
    ex = backend.onCreate([xin], [yout], op)
    assert ex is not None and ex.onResize([xin], [yout]) == 0
    assert yout.shape == (n, oc, 18, 18)
    backend.onAcquire(yout)
    yout.data.fill_(float("nan"))
    assert ex.onExecute([xin], [yout]) == 0
    backend.onSync()
    ref, _ = deconv_f32(x, w, b, 2, 1, 1, 2, depthwise=dw)
    assert rel_err(backend.onCopyBuffer(yout, "same"), ref) <= 1e-4


@pytest.mark.parametrize("name", list(G.CASES))
def test_deconv_f32_matches_reference_golden(backend, name):
    """every recorded case of tests/golden/deconv_f32_golden.npz (outputs of the reference CPU backend) within 1e-3 of max|y|,
    resized the way the plugin resizes: begin pads from convolutionTransposePad and the output size from shape inference"""
    golden = G.load()
    n, ic, oc, hw, k, s, pads, d, op, same, out, dw, relu, relu6 = G.CASES[name]
    x, w, b = G.case_inputs(name)
    a = 2 if relu6 else relu
    shape = golden[name][2]
    pad = G.begin_pads(name, shape[2:])
    h = create(backend, ic, oc, k, s, 0, d, a, w, b, depthwise=bool(dw))
    try:
        assert dlib().mnnb200_deconv_f32_set_pad(h, *pad) == 0
        assert resize(h, n, hw, out=shape[2:], depthwise=bool(dw)) == shape[2:]
        f = dlib().mnnb200_dwdeconv_f32_execute if dw else dlib().mnnb200_deconv_f32_execute
        y = execute_with(backend, f, h, x, shape).cpu().numpy()
        err = golden_check(y, name, golden, 1e-3)
        print(f"{name}: rel err {err:.2e} against the reference CPU")
    finally:
        lib().mnnb200_exec_destroy(h)
