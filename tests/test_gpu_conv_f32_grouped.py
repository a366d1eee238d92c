"""Grouped fp32 convolution through the C ABI (-m gpu): mnnb200_conv_f32_create_grouped on the split-TF32 wgmma conv kernel,
against float64 torch on the CPU.

Every output must lie within the split-TF32 error model (tests/test_gpu_conv_f32.py::conv_tolerance) at the n chunk's K (the
block-diagonal zeros add exact zeros), and all of them within 1e-4 of max|ref|.  Inputs and outputs sit between NaN guard bands,
4 bytes past 16-byte alignment.  Each case reads back its plan through mnnb200_conv_f32_plan: tile width, n chunks, whole groups
per chunk P, chunks per group Q and the chunk's padded input channels cp8."""
import ctypes as C

import numpy as np
import pytest

from tests.golden import make_gconv_golden as GG
from tests.test_gconv_cpu import chunk_plan
from tests.test_gpu_conv_f32 import (INVALID_VALUE, NO_EXECUTION, NOT_SUPPORT, check_elements, conv64, conv_tolerance, desc,
                                     execute, image_for_tiles, lib, natural_out, pair, plan_bn, rel_err, sm_count)

pytestmark = pytest.mark.gpu

PLAN9 = ("bn", "n_chunks", "m_tiles", "num_kb", "stages", "cp8", "taps", "P", "Q")


def plan9(h):
    f = (C.c_int * 9)(*([-7] * 9))
    assert lib().mnnb200_conv_f32_plan(h, f, 9) == 0, lib().mnnb200_last_error()
    return dict(zip(PLAN9, f))


def inputs(rng, n, ic, oc, group, k, hw, wscale=1.0):
    (kh, kw), (ih, iw) = pair(k), pair(hw)
    x = rng.standard_normal((n, ic, ih, iw)).astype(np.float32)
    fan = ic // group * kh * kw
    w = (rng.uniform(-1, 1, (oc, ic // group, kh, kw)) * 1.2 * wscale / np.sqrt(fan)).astype(np.float32)
    b = rng.uniform(-0.5, 0.5, oc).astype(np.float32)
    return x, w, b


def create(backend, ic, oc, group, k, s, p, d, a, w, b, grouped=True):
    h = C.c_void_p()
    dd = desc(ic, oc, k, s, p, d, group, int(a >= 1))
    f = lib().mnnb200_conv_f32_create_grouped if grouped else lib().mnnb200_conv_f32_create
    st = f(backend.runtime._h, C.byref(dd), w.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), int(a == 2), C.byref(h))
    assert st == 0, lib().mnnb200_last_error()
    return h


def resize(h, n, hw, out=None):
    (ih, iw), (oh0, ow0) = pair(hw), out or (0, 0)
    oh, ow = C.c_int(oh0), C.c_int(ow0)
    assert lib().mnnb200_conv_f32_resize(h, n, ih, iw, C.byref(oh), C.byref(ow)) == 0, lib().mnnb200_last_error()
    return oh.value, ow.value


def run(backend, h, x, w, b, group, s, p, d, a, out_hw, what):
    """execute the resized grouped conv h on x (guarded) and check every output: (rel err, plan, y, ref)"""
    pl = plan9(h)
    n, oc = x.shape[0], w.shape[0]
    y = execute(backend, h, x, (n, oc) + tuple(out_hw)).cpu().numpy()
    ref, S = conv64(x, w, b, s, p, d, a, groups=group, out_hw=tuple(out_hw))
    check_elements(y, ref, conv_tolerance(S, b, pl["num_kb"] * 32), what)
    err = rel_err(y, ref)
    assert err <= 1e-4, f"{what}: split-TF32 rel err {err:.2e}"
    return err, pl, y, ref


def expected_plan(group, ic, oc):
    """(bn, P, Q, n_chunks, cp8) of capi.cu conv_f32_create for group > 1"""
    return chunk_plan(group, ic // group, oc // group)


# name: ic, oc, group, kernel, stride, pad, dilation, (ih, iw), batch, act
CASES = {
    "P8_G13_not_multiple": (52, 52, 13, 3, 1, 1, 1, (10, 9), 2, 1),
    "Q2_ocg160_ragged": (15, 480, 3, 3, 1, 1, 1, (7, 8), 2, 0),
    "icg1_ocg2": (24, 48, 24, 3, 1, 1, 1, (9, 11), 2, 2),
    "icg3_ocg8": (24, 64, 8, 3, 1, 1, 1, (12, 10), 2, 1),
    "icg5_ocg40": (20, 160, 4, 3, 2, 1, 1, (13, 12), 2, 0),
    "icg12_ocg16": (72, 96, 6, 3, 1, 1, 1, (8, 9), 2, 1),
    "ring_wraps_icg32": (128, 128, 4, 3, 1, 1, 1, (9, 7), 2, 1),
    "k3x5_s2x1_d2x1_nonsquare": (32, 64, 4, (3, 5), (2, 1), (2, 2), (2, 1), (15, 11), 2, 0),
    "k5_s2_d2": (48, 96, 3, 5, 2, 4, 2, (17, 19), 2, 1),
    "relu6_clamps": (40, 80, 5, 3, 1, 1, 1, (9, 9), 2, 2),
    "depthwise_shape_g24": (24, 24, 24, 3, 1, 1, 1, (10, 12), 2, 1),
    "shufflenet_g3_1x1": (240, 240, 3, 1, 1, 0, 1, (14, 14), 4, 1),
    "alexnet_g2_k5": (96, 256, 2, 5, 1, 2, 1, (13, 13), 2, 1),
}


@pytest.mark.parametrize("name", list(CASES))
def test_grouped_conv_matches_float64(backend, name):
    ic, oc, group, k, s, p, d, hw, n, a = CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    x, w, b = inputs(rng, n, ic, oc, group, k, hw, wscale=8 if name == "relu6_clamps" else 1)
    h = create(backend, ic, oc, group, k, s, p, d, a, w, b)
    try:
        oh, ow = resize(h, n, hw)
        (kh, kw), (sh, sw), (ph, pw), (dh, dw) = pair(k), pair(s), pair(p), pair(d)
        assert (oh, ow) == (natural_out(hw[0], kh, sh, ph, dh), natural_out(hw[1], kw, sw, pw, dw))
        err, pl, _, ref = run(backend, h, x, w, b, group, s, p, d, a, (oh, ow), name)
        bn, P, Q, chunks, cp8 = expected_plan(group, ic, oc)
        assert (pl["bn"], pl["P"], pl["Q"], pl["n_chunks"], pl["cp8"], pl["taps"]) == (bn, P, Q, chunks, cp8, kh * kw), pl
        assert pl["num_kb"] == -(-kh * kw * cp8 // 32)
        if name == "P8_G13_not_multiple":
            assert P == 8 and group % P
        if name == "Q2_ocg160_ragged":
            assert Q == 2 and (oc // group) % bn
        if name == "ring_wraps_icg32":
            assert pl["num_kb"] > pl["stages"] and pl["num_kb"] % pl["stages"], pl
        if name == "relu6_clamps":
            assert (ref == 6).any() and (ref == 0).any()
        bm, macs = C.c_double(), C.c_double()
        assert lib().mnnb200_exec_cost(h, C.byref(bm), C.byref(macs)) == 0
        assert macs.value == n * oh * ow * oc * (ic // group) * kh * kw
        print(f"{name}: plan {pl}, rel err {err:.2e}")
    finally:
        lib().mnnb200_exec_destroy(h)


def test_grouped_conv_items_past_the_sms(backend):
    """more work items than SMs, an n chunk count that does not divide the grid (a CTA's items change chunk), an M tile across two
    images and a part-empty last M tile"""
    sms = sm_count()
    ic, oc, group, a = 160, 160, 40, 1                 # icg = ocg = 4: P = 8, 5 n chunks
    chunks = expected_plan(group, ic, oc)[3]
    assert sms % chunks
    m = sms // chunks + 3
    n = 2
    hw = image_for_tiles(m, n)
    rng = np.random.default_rng(11)
    x, w, b = inputs(rng, n, ic, oc, group, 3, hw)
    h = create(backend, ic, oc, group, 3, 1, 1, 1, a, w, b)
    try:
        oh, ow = resize(h, n, hw)
        err, pl, _, _ = run(backend, h, x, w, b, group, 1, 1, 1, a, (oh, ow), "items past the SMs")
        assert pl["m_tiles"] * pl["n_chunks"] > sms and pl["n_chunks"] == chunks
        assert (oh * ow) % 128 and (n * oh * ow) % 128
        print(f"items past the SMs: plan {pl}, {pl['m_tiles'] * pl['n_chunks']} items on {sms} SMs, rel err {err:.2e}")
    finally:
        lib().mnnb200_exec_destroy(h)


def test_grouped_conv_set_pad_asymmetric(backend):
    """begin pads set after create with an explicit output larger than the natural one: effective pads [t, l, b, r] differ"""
    ic, oc, group, n, (ih, iw) = 24, 48, 3, 2, (15, 20)
    rng = np.random.default_rng(12)
    x, w, b = inputs(rng, n, ic, oc, group, 3, (ih, iw))
    h = create(backend, ic, oc, group, 3, 2, 0, 1, 1, w, b)
    try:
        assert lib().mnnb200_conv_f32_set_pad(h, 1, 0) == 0
        assert resize(h, n, (ih, iw), out=(8, 10)) == (8, 10)
        run(backend, h, x, w, b, group, 2, (1, 0), 1, 1, (8, 10), "set_pad asymmetric")
    finally:
        lib().mnnb200_exec_destroy(h)


def test_grouped_conv_re_resize_keeps_width(backend):
    """one execution resized batch 1 -> a shape with many M tiles -> new pads -> batch 1: the width fixed at create is kept (a
    group-1 conv of these channels would plan 32 and 128)"""
    sms = sm_count()
    ic, oc, group, a = 64, 256, 2, 1                   # ocg 128: bn 128
    rng = np.random.default_rng(13)
    _, w, b = inputs(rng, 1, ic, oc, group, 3, 1)
    h = create(backend, ic, oc, group, 3, 1, 1, 1, a, w, b)
    m128 = next(m for m in range(1, 4 * sms) if plan_bn(oc, m, sms) == 128)
    try:
        seen = []
        for n, hw, pad in ((1, (9, 11), (1, 1)), (2, image_for_tiles(m128), (1, 1)), (1, (10, 7), (0, 2))):
            if pad != (1, 1):
                assert lib().mnnb200_conv_f32_set_pad(h, *pad) == 0
            x = rng.standard_normal((n, ic) + hw).astype(np.float32)
            oh, ow = resize(h, n, hw)
            _, pl, _, _ = run(backend, h, x, w, b, group, 1, pad, 1, a, (oh, ow), f"resize to {n} x {hw}")
            seen.append((pl["bn"], pl["n_chunks"], pl["P"], pl["Q"]))
        assert seen == [(128, 2, 1, 1)] * 3
        assert plan_bn(oc, 1, sms) == 32
    finally:
        lib().mnnb200_exec_destroy(h)


@pytest.mark.parametrize("bn", [32, 64, 128])
def test_group1_through_create_grouped_is_bit_identical(backend, bn):
    """group 1 through create_grouped gives the execution conv_f32_create gives: the same plan and the same output bits"""
    import torch
    sms = sm_count()
    ic, oc, k, a = 40, {32: 24, 64: 56, 128: 200}[bn], 3, 1
    m = next(m for m in range(1, 4 * sms) if plan_bn(oc, m, sms) == bn)
    n = 2
    hw = image_for_tiles(m, n)
    rng = np.random.default_rng(bn)
    x, w, b = inputs(rng, n, ic, oc, 1, k, hw)
    hs = [create(backend, ic, oc, 1, k, 1, 1, 1, a, w, b, grouped=g) for g in (False, True)]
    try:
        outs = []
        for h in hs:
            oh, ow = resize(h, n, hw)
            outs.append((plan9(h), execute(backend, h, x, (n, oc, oh, ow)).cpu()))
        (p0, y0), (p1, y1) = outs
        assert p0 == p1 and p0["bn"] == bn and (p0["P"], p0["Q"]) == (1, p0["n_chunks"])
        assert torch.equal(y0.view(torch.int32), y1.view(torch.int32))
    finally:
        for h in hs:
            lib().mnnb200_exec_destroy(h)


@pytest.mark.parametrize("name", list(GG.CASES))
def test_golden_cases_within_1e3_of_cpu(backend, name):
    """every recorded case of the reference CPU (tests/golden/gconv_f32_golden.npz) through create_grouped, with the group the
    CPU takes from inputCount: within 1e-3 of the CPU's outputs and within the error model of float64"""
    from oracle import gconv_oracle as D
    n, ic, oc, hw, k, s, pads, d, group, input_count, relu, relu6 = GG.CASES[name]
    rec, idx, shape = GG.load()[name]
    g = D.cpu_group(group, input_count, ic)
    x, w, b = GG.case_inputs(name)
    a = 2 if relu6 else relu
    h = create(backend, ic, oc, g, k, s, (pads[0], pads[1]), d, a, w, b)
    try:
        oh, ow = resize(h, n, hw, out=tuple(shape[2:]))
        err, _, y, _ = run(backend, h, x, w, b, g, s, (pads[0], pads[1]), d, a, (oh, ow), name)
        flat = y.astype(np.float64).reshape(-1)
        got = flat if idx is None else flat[idx]
        cpu_err = float(np.abs(got - rec).max() / max(np.abs(rec).max(), 1e-30))
        assert cpu_err <= 1e-3, f"{name}: {cpu_err:.2e} from the reference CPU"
        print(f"{name}: {cpu_err:.2e} from the reference CPU, {err:.2e} from float64")
    finally:
        lib().mnnb200_exec_destroy(h)


def test_grouped_refusals_keep_the_plan(backend):
    """create_grouped refuses NULL arguments and bad descriptors (INVALID_VALUE) and a group that does not divide ic or oc
    (NOT_SUPPORT), conv_f32_create still refuses group 2, and a refused resize keeps the previous plan: after each refusal the
    resized execution still computes its conv"""
    ic, oc, group, n, hw = 24, 48, 3, 2, (9, 10)
    rng = np.random.default_rng(14)
    x, w, b = inputs(rng, n, ic, oc, group, 3, hw)
    h = create(backend, ic, oc, group, 3, 1, 1, 1, 1, w, b)
    rt, L = backend.runtime._h, lib()
    wp = w.ctypes.data_as(C.c_void_p)
    try:
        f = (C.c_int * 9)()
        assert L.mnnb200_conv_f32_plan(h, f, 9) == NO_EXECUTION
        oh, ow = resize(h, n, hw)
        before = plan9(h)
        run(backend, h, x, w, b, group, 1, 1, 1, 1, (oh, ow), "before the refusals")
        refused = []
        for what, dd, r_, weights, want in (
                ("NULL runtime", desc(ic, oc, 3, 1, 1, 1, group, 1), None, wp, INVALID_VALUE),
                ("NULL weights", desc(ic, oc, 3, 1, 1, 1, group, 1), rt, None, INVALID_VALUE),
                ("group 0", desc(ic, oc, 3, 1, 1, 1, 0, 1), rt, wp, INVALID_VALUE),
                ("stride 0", desc(ic, oc, 3, 0, 1, 1, group, 1), rt, wp, INVALID_VALUE),
                ("group 5 of ic 24", desc(ic, 40, 3, 1, 1, 1, 5, 1), rt, wp, NOT_SUPPORT),
                ("group 4 of oc 42", desc(ic, 42, 3, 1, 1, 1, 4, 1), rt, wp, NOT_SUPPORT)):
            out = C.c_void_p()
            assert L.mnnb200_conv_f32_create_grouped(r_, C.byref(dd), weights, None, 0, C.byref(out)) == want, what
            assert not out.value, what
            refused.append(what)
        out = C.c_void_p()
        assert L.mnnb200_conv_f32_create_grouped(rt, None, wp, None, 0, C.byref(out)) == INVALID_VALUE
        assert L.mnnb200_conv_f32_create(rt, C.byref(desc(ic, oc, 3, 1, 1, 1, group, 1)), wp, None, 0, C.byref(out)) == NOT_SUPPORT
        assert not out.value
        o, p = C.c_int(0), C.c_int(0)
        assert L.mnnb200_conv_f32_resize(h, 2 ** 20, 2 ** 10, 2 ** 10, C.byref(o), C.byref(p)) == NOT_SUPPORT
        assert L.mnnb200_conv_f32_plan(h, f, 7) == 0 and list(f)[:7] == [before[k] for k in PLAN9[:7]]
        assert plan9(h) == before
        run(backend, h, x, w, b, group, 1, 1, 1, 1, (oh, ow), "after the refusals")
        print("refused:", ", ".join(refused))
    finally:
        L.mnnb200_exec_destroy(h)


def test_grouped_through_backend_mirror(backend):
    """Backend.onCreate -> onResize -> onExecute for a grouped Convolution of the Python mirror; weights not shaped
    [oc][ic/group][kh][kw] are not taken"""
    from mnn_b200.backend import Op, Tensor
    n, ic, oc, group, hw = 2, 32, 64, 8, 11
    rng = np.random.default_rng(15)
    x, w, b = inputs(rng, n, ic, oc, group, 3, hw)
    op = Op(type="Convolution", conv=dict(ic=ic, oc=oc, kernel=(3, 3), stride=(2, 2), pad=(1, 1), group=group, relu=True),
            weight=w, bias=b, relu6=False)
    xin = backend.onAcquire(Tensor((n, ic, hw, hw), "float"))
    backend.onCopyBuffer(x, xin)
    yout = Tensor((n, oc, 1, 1), "float")
    ex = backend.onCreate([xin], [yout], op)
    assert ex is not None and ex.onResize([xin], [yout]) == 0
    assert yout.shape == (n, oc, 6, 6)
    backend.onAcquire(yout)
    yout.data.fill_(float("nan"))
    assert ex.onExecute([xin], [yout]) == 0
    backend.onSync()
    ref, _ = conv64(x, w, b, 2, 1, 1, 1, groups=group)
    assert rel_err(backend.onCopyBuffer(yout, "same"), ref) <= 1e-4
    wrong = Op(type="Convolution", conv=dict(ic=ic, oc=oc, kernel=(3, 3), group=4), weight=w, bias=b)
    assert backend.onCreate([xin], [yout], wrong) is None
