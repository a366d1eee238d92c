"""fp32 convolution and its fp32 neighbours through the C ABI (-m gpu), against float64 torch on the CPU.

Every output of the split-TF32 conv (a_hi*w_hi + a_hi*w_lo + a_lo*w_hi, fp32 accumulate) must lie within a worst-case error
model of that arithmetic (conv_tolerance), and all of them together within 1e-4 of max|ref| (the ABI's accuracy contract); every
output of the depthwise conv within the model of its fmaf chain (dw_tolerance) and 1e-5 of max|ref|; add and scale within 1e-5,
softmax within 1e-4.  A conv's input sits in a larger buffer between NaN guard bands, 4 bytes past 16-byte alignment, and its
output in a NaN-filled buffer: a read outside x turns an output NaN, and a write outside y or an output left unwritten shows.
The conv cases read back through mnnb200_conv_f32_plan which tile width and pipeline cell resize gave them; the cell matrix and the
probes derive their shapes from the SM count with resize's own rule (plan_bn).  Two layers also report what plain TF32 (inputs and
weights rounded to a 10-bit mantissa) would give."""
import ctypes as C
import functools
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NOT_SUPPORT, NO_EXECUTION, INVALID_VALUE = 2, 4, 5
GUARD = 4097                 # NaN floats either side of a conv's x and y; 4097 * 4 bytes puts the tensors 4 bytes past 16-byte alignment
PLAN_FIELDS = ("bn", "n_chunks", "m_tiles", "num_kb", "stages", "cp8", "taps")

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


def pair(v):
    return tuple(v) if isinstance(v, (tuple, list)) else (v, v)


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


def natural_out(i, k, s, p, d):
    return (i + 2 * p - d * (k - 1) - 1) // s + 1


def conv64(x, w, b, stride, pad, dil, a, groups=1, out_hw=None):
    """float64 (ref, S) on the CPU.  ref = act(conv(x, w) + b) with begin pads `pad` and output size out_hw (natural when None):
    zeros after the input as far as the output reaches, which is what the kernels read for out-of-image taps.  S = conv(|x|, |w|)
    over the same window, no bias: the magnitude sum the error models scale with."""
    import torch
    import torch.nn.functional as F
    x = (x if isinstance(x, torch.Tensor) else torch.from_numpy(np.asarray(x))).to("cpu", torch.float64)
    w = torch.from_numpy(np.asarray(w, np.float64))
    (sh, sw), (ph, pw), (dh, dw) = pair(stride), pair(pad), pair(dil)
    ih, iw = x.shape[2:]
    kh, kw = w.shape[2:]
    oh, ow = out_hw or (natural_out(ih, kh, sh, ph, dh), natural_out(iw, kw, sw, pw, dw))
    eh, ew = max(0, (oh - 1) * sh + dh * (kh - 1) + 1 - ih - ph), max(0, (ow - 1) * sw + dw * (kw - 1) + 1 - iw - pw)
    xp = F.pad(x, (pw, ew, ph, eh))

    def conv(xx, ww):
        return F.conv2d(xx, ww, None, (sh, sw), 0, (dh, dw), groups)[:, :, :oh, :ow]

    y = conv(xp, w) + torch.from_numpy(np.asarray(b, np.float64))[None, :, None, None]
    assert tuple(y.shape[2:]) == (oh, ow)
    return act(y, a).numpy(), conv(xp.abs(), w.abs()).numpy()


def conv_ref(x, w, b, stride, pad, dil, a, groups=1):
    return conv64(x, w, b, stride, pad, dil, a, groups)[0]


# Worst-case model of the split-TF32 conv, per output element (the tf32 GEMM's model in tests/test_matmul.py::tolerance, split):
# an fp32 value a is split into a_hi = tf32(a) and a_lo = tf32(a - a_hi); |a - a_hi| <= 2^-11 |a| (a - a_hi is exact in fp32)
# and rounding it to TF32 errs by <= 2^-11 |a - a_hi| <= 2^-22 |a|; the same for w.  Products of TF32 values are exact in fp32,
# so a_hi w_hi + a_hi w_lo + a_lo w_hi misses a w only by the dropped a_lo w_lo and the two low parts' roundings, about
# 3 2^-22 |a||w| together: under 2^-20 |a||w| per product, 2^-20 S in all, S = conv(|x|, |w|).  The accumulation is
# 3 ceil(Kp / 8) wgmma k8 steps (Kp = num_kb * 32, padded channels and taps included); each aligns its 8 products and the
# accumulator to the largest exponent and truncates, then truncates the normalised sum, so it errs by at most (8 + 2) 2^-23 of
# its terms' magnitude sum, which S bounds.  The epilogue's bias add rounds once, <= 2^-24 |acc + bias|, which
# 2^-23 (S + |bias|) covers.  ReLU and ReLU6 are 1-Lipschitz, so the bound holds after them.  At Kp = 64 that is about 3e-5 S.
def conv_tolerance(s, bias, kp):
    tau = 2.0 ** -20 + 3 * -(-kp // 8) * (8 + 2) * 2.0 ** -23
    return tau * s + 2.0 ** -23 * (s + np.abs(np.asarray(bias, np.float64))[None, :, None, None])


# The depthwise kernel is one fmaf chain per output over its in-image taps: each fma rounds once, by <= 2^-24 of the running
# sum, which S bounds; then one rounded bias add.  ReLU / ReLU6 as above.
def dw_tolerance(s, bias, taps):
    return taps * 2.0 ** -24 * s + 2.0 ** -23 * (s + np.abs(np.asarray(bias, np.float64))[None, :, None, None])


def check_elements(y, ref, tol, what):
    y = np.asarray(y, np.float64)
    assert y.shape == ref.shape, (y.shape, ref.shape)
    assert np.isfinite(y).all(), f"{what}: {np.count_nonzero(~np.isfinite(y))} outputs not finite"
    over = np.abs(y - ref) > tol
    if over.any():
        i = tuple(np.argwhere(over)[0])
        raise AssertionError(f"{what}: {over.sum()} of {over.size} outputs outside the error bound; first at (n, c, h, w) {i}: "
                             f"y {y[i]!r}, float64 {ref[i]!r}, bound {tol[i]:.3g}")


def conv_inputs(rng, ic, oc, k, hw, n, depthwise=False):
    (kh, kw), (ih, iw) = pair(k), pair(hw)
    x = rng.standard_normal((n, ic, ih, iw)).astype(np.float32)
    ks = (1 if depthwise else ic) * kh * kw
    w = (rng.uniform(-1, 1, (oc, 1 if depthwise else ic, kh, kw)) * 1.2 / np.sqrt(ks)).astype(np.float32)
    b = rng.uniform(-0.5, 0.5, oc).astype(np.float32)
    return x, w, b


def desc(ic, oc, k, s, p, d, group, relu):
    from mnn_b200._capi import ConvDesc
    (kh, kw), (sh, sw), (ph, pw), (dh, dw) = pair(k), pair(s), pair(p), pair(d)
    return ConvDesc(ic, oc, kh, kw, sh, sw, ph, pw, dh, dw, group, relu)


def create_conv(backend, ic, oc, k, s, p, d, a, w, b, depthwise=False):
    h = C.c_void_p()
    f = lib().mnnb200_dwconv_f32_create if depthwise else lib().mnnb200_conv_f32_create
    dd = desc(ic, oc, k, s, p, d, ic if depthwise else 1, int(a >= 1))
    st = f(backend.runtime._h, C.byref(dd), w.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), int(a == 2), C.byref(h))
    assert st == 0, lib().mnnb200_last_error()
    return h


def resize(h, n, hw, depthwise=False, out=None):
    """hw: input h = w, or (ih, iw); out: an explicit (oh, ow) as the plugin passes for TF-SAME padding"""
    (ih, iw), (oh0, ow0) = pair(hw), out or (0, 0)
    oh, ow = C.c_int(oh0), C.c_int(ow0)
    f = lib().mnnb200_dwconv_f32_resize if depthwise else lib().mnnb200_conv_f32_resize
    assert f(h, n, ih, iw, C.byref(oh), C.byref(ow)) == 0, lib().mnnb200_last_error()
    return oh.value, ow.value


def plan(h):
    f = (C.c_int * len(PLAN_FIELDS))()
    assert lib().mnnb200_conv_f32_plan(h, f, len(f)) == 0, lib().mnnb200_last_error()
    return dict(zip(PLAN_FIELDS, f))


def guarded(shape, fill=None):
    """(buffer, view): a `shape` view GUARD floats into a NaN-filled fp32 buffer GUARD floats longer on each side; fill (host
    array or tensor) is copied into the view"""
    import torch
    count = int(np.prod(shape))
    buf = torch.full((count + 2 * GUARD,), float("nan"), dtype=torch.float32, device="cuda")
    view = buf[GUARD:GUARD + count].view(tuple(shape))
    assert view.data_ptr() % 16 == 4
    if fill is not None:
        view.copy_(fill if isinstance(fill, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(fill, np.float32)))
    return buf, view


def execute(backend, h, x, out_shape, depthwise=False):
    """run a resized conv / depthwise execution on x with both tensors guarded; the device output after checking the guards"""
    import torch
    xb, xd = guarded(x.shape, x)
    yb, yd = guarded(out_shape)
    f = lib().mnnb200_dwconv_f32_execute if depthwise else lib().mnnb200_conv_f32_execute
    assert f(h, ptr(xd), ptr(yd)) == 0, lib().mnnb200_last_error()
    backend.onSync()
    for buf, t, what in ((xb, xd, "x"), (yb, yd, "y")):
        g = torch.cat([buf[:GUARD], buf[GUARD + t.numel():]])
        assert bool(torch.isnan(g).all()), f"{int((~torch.isnan(g)).sum())} floats of {what}'s guard bands were written"
    return yd


def run_conv(backend, h, x, w, b, s, p, d, a, out_hw, images=None, what=""):
    """execute the resized conv h on x and check images `images` (all by default) per element against float64 and by the
    max-norm contract: (max|y - ref| / max|ref|, plan, ref, S, y)"""
    pl = plan(h)
    n, oc = x.shape[0], w.shape[0]
    yd = execute(backend, h, x, (n, oc) + tuple(out_hw))
    idx = list(range(n)) if images is None else list(images)
    y = yd[idx].cpu().numpy()
    ref, S = conv64(x[idx], w, b, s, p, d, a, out_hw=tuple(out_hw))
    check_elements(y, ref, conv_tolerance(S, b, pl["num_kb"] * 32), what)
    err = rel_err(y, ref)
    assert err <= 1e-4, f"{what}: split-TF32 rel err {err:.2e}"
    return err, pl, ref, S, y


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def plan_bn(oc, m_tiles, sms):
    """capi.cu mnnb200_conv_f32_resize: the widest tile oc wants, halved while the work items would not fill the SMs"""
    bn = 32 if oc <= 32 else 64 if oc <= 64 else 128
    while bn > 32 and m_tiles * -(-oc // bn) < sms:
        bn //= 2
    return bn


def image_for_tiles(m, n=2, w=13):
    """(h, w) of n images whose n*h*w output pixels fill m 128-row M tiles, the last one part empty, and an M tile that spans
    two images"""
    for h in range((m - 1) * 128 // (n * w) + 1, m * 128 // (n * w) + 1):
        if (m - 1) * 128 < n * h * w < m * 128 and (h * w) % 128:
            return h, w
    raise AssertionError(f"no {n} images of width {w} fill {m} M tiles")


@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: "ic%d_oc%d_k%d_s%d_p%d_d%d_hw%d_n%d_a%d" % c)
def test_conv_f32_matches_float64(backend, case):
    ic, oc, k, s, p, d, hw, n, a = case
    rng = np.random.default_rng(ic * 131 + oc + k)
    x, w, b = conv_inputs(rng, ic, oc, k, hw, n)
    h = create_conv(backend, ic, oc, k, s, p, d, a, w, b)
    try:
        oh, ow = resize(h, n, hw)
        assert (oh, ow) == (natural_out(hw, k, s, p, d),) * 2
        err, pl, ref, _, _ = run_conv(backend, h, x, w, b, s, p, d, a, (oh, ow), what="conv")
        msg = f"split-TF32 rel err {err:.2e}, plan {pl}"
        if CONV_CASES.index(case) in TF32_REPORT:
            msg += f", plain TF32 would give {rel_err(conv_ref(tf32(x), tf32(w), b, s, p, d, a), ref):.2e}"
        print(msg)
        bm, macs = C.c_double(), C.c_double()
        assert lib().mnnb200_exec_cost(h, C.byref(bm), C.byref(macs)) == 0
        assert macs.value == n * oh * ow * oc * ic * k * k
    finally:
        lib().mnnb200_exec_destroy(h)


# name: ic, oc, kernel, stride, pad, dilation, (ih, iw), batch, act.  ic 1 / 5 (cp8 8: a K block spans 4 taps), 13 (cp8 16: 2 taps)
# and 40 (cp8 40: a K block holds part of a tap); "beyond" pads reach past the kernel, so whole output rows / columns are bias only
GEOMETRY = {
    "k1x7_p0x3_ic40": (40, 48, (1, 7), 1, (0, 3), 1, (17, 17), 2, 1),
    "k7x1_p3x0_ic40": (40, 48, (7, 1), 1, (3, 0), 1, (17, 17), 2, 1),
    "k3x1_p1x0_ic13": (13, 24, (3, 1), 1, (1, 0), 1, (15, 11), 2, 0),
    "s1x2_ic5": (5, 20, 3, (1, 2), 1, 1, (19, 23), 2, 0),
    "s2x1_ic13": (13, 36, 3, (2, 1), 1, 1, (21, 14), 2, 1),
    "p0x2_ic13": (13, 40, 3, 1, (0, 2), 1, (12, 9), 3, 0),
    "d1x2_p1x2": (16, 40, 3, 1, (1, 2), (1, 2), (13, 15), 2, 0),
    "d3x1_p3x1": (8, 24, 3, 1, (3, 1), (3, 1), (16, 12), 2, 1),
    "ih27_iw45_s2_ic1": (1, 33, 3, 2, 1, 1, (27, 45), 2, 1),
    "k11_s4_ic3": (3, 64, 11, 4, 2, 1, (63, 67), 2, 1),
    "beyond_p4x1_none": (5, 24, 3, 1, (4, 1), 1, (6, 9), 2, 0),
    "beyond_p2x5_relu6": (5, 24, (1, 3), 1, (2, 5), 1, (7, 4), 2, 2),
    "relu6_both_clamps": (13, 32, 3, 1, 1, 1, (14, 10), 2, 2),
}


@pytest.mark.parametrize("name", list(GEOMETRY))
def test_conv_f32_geometry(backend, name):
    import torch
    ic, oc, k, s, p, d, hw, n, a = GEOMETRY[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    x, w, b = conv_inputs(rng, ic, oc, k, hw, n)
    if name.startswith("beyond") and a == 2:
        b = rng.uniform(0.5, 8, oc).astype(np.float32)          # bias-only outputs in (0, 6] after ReLU6
    if name == "relu6_both_clamps":
        w *= 8
    h = create_conv(backend, ic, oc, k, s, p, d, a, w, b)
    try:
        oh, ow = resize(h, n, hw)
        (kh, kw), (sh, sw), (ph, pw), (dh, dw) = pair(k), pair(s), pair(p), pair(d)
        assert (oh, ow) == (natural_out(hw[0], kh, sh, ph, dh), natural_out(hw[1], kw, sw, pw, dw))
        err, pl, ref, S, _ = run_conv(backend, h, x, w, b, s, p, d, a, (oh, ow), what=name)
        assert (pl["cp8"], pl["taps"]) == (-(-ic // 8) * 8, kh * kw)
        print(f"{name}: split-TF32 rel err {err:.2e}, plan {pl}")
        if name.startswith("beyond"):
            bias_only = (S == 0).all(axis=(0, 1))
            assert bias_only.all(axis=1).any() and bias_only[0].all(), "wanted whole output rows that are bias only"
            if pw > kw:
                assert bias_only.all(axis=0).any(), "wanted whole output columns that are bias only"
            expect = act(torch.from_numpy(b.astype(np.float64)), a).numpy()
            assert (expect != 0).all()
            assert np.array_equal(ref[:, :, bias_only], np.broadcast_to(expect[None, :, None], ref[:, :, bias_only].shape))
        if name == "relu6_both_clamps":
            assert (ref == 6).any() and (ref == 0).any() and ((ref > 0) & (ref < 6)).any()
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
        assert resize(h, n, hw, out=(7, 7)) == (7, 7)
        xpad = np.pad(x, ((0, 0), (0, 0), (0, 1), (0, 1)))
        ref = conv_ref(xpad, w, b, s, 0, 1, 0)
        assert ref.shape == (n, oc, 7, 7)
        _, _, ref2, _, _ = run_conv(backend, h, x, w, b, s, 0, 1, 0, (7, 7), what="set_pad")
        assert np.array_equal(ref, ref2)
    finally:
        lib().mnnb200_exec_destroy(h)


def test_conv_f32_set_pad_non_square(backend):
    """set_pad with pad_h != pad_w and an explicit output wider than the natural one (TF-SAME, stride 2, even iw)"""
    ic, oc, n, (ih, iw) = 12, 20, 2, (15, 20)
    rng = np.random.default_rng(9)
    x, w, b = conv_inputs(rng, ic, oc, 3, (ih, iw), n)
    h = create_conv(backend, ic, oc, 3, 2, 0, 1, 1, w, b)
    try:
        assert lib().mnnb200_conv_f32_set_pad(h, 1, 0) == 0
        assert natural_out(iw, 3, 2, 0, 1) == 9
        assert resize(h, n, (ih, iw), out=(8, 10)) == (8, 10)
        xpad = np.pad(x, ((0, 0), (0, 0), (1, 1), (0, 1)))
        ref = conv_ref(xpad, w, b, 2, 0, 1, 1)
        assert ref.shape == (n, oc, 8, 10)
        _, _, ref2, _, _ = run_conv(backend, h, x, w, b, 2, (1, 0), 1, 1, (8, 10), what="set_pad non-square")
        assert np.array_equal(ref, ref2)
    finally:
        lib().mnnb200_exec_destroy(h)


def cell_shape(bn, sms):
    """(oc, m_tiles) that resize plans at width bn with more work items than SMs, a ragged last n chunk, and a chunk count that
    does not divide the grid, so that consecutive items of a CTA fall in different n chunks"""
    for chunks in range(2, 64):
        if sms % chunks:
            oc = bn * (chunks - 1) + bn // 2 + 3
            lo = sms // chunks + 1
            ms = [m for m in range(lo, 2 * lo) if plan_bn(oc, m, sms) == bn]
            if ms:
                return oc, ms[-1]
    raise AssertionError(f"no multi-item shape at width {bn} for {sms} SMs")


# name: (ic, kernel, pad, act).  kb1: 1x1, ic 20 (padded to 24), one K block; kb9: 3x3, ic 31, K = 288 = 9 blocks, more than
# any width's ring holds and not a multiple of it, so the ring wraps inside an item and its phase carries into the next item
CELLS = {"kb1": (20, 1, 0, 2), "kb9": (31, 3, 1, 1)}


@pytest.mark.parametrize("bn", [32, 64, 128])
@pytest.mark.parametrize("cell", list(CELLS))
def test_conv_f32_cell_matrix(backend, bn, cell):
    """each tile width with one K block and with a wrapping ring, both with several items per CTA whose n chunk changes from
    item to item, a ragged last n chunk, an M tile across two images and a part-empty last M tile"""
    sms = sm_count()
    ic, k, p, a = CELLS[cell]
    oc, m = cell_shape(bn, sms)
    n = 2
    hw = image_for_tiles(m, n)
    rng = np.random.default_rng(bn * 10 + k)
    x, w, b = conv_inputs(rng, ic, oc, k, hw, n)
    h = create_conv(backend, ic, oc, k, 1, p, 1, a, w, b)
    try:
        oh, ow = resize(h, n, hw)
        err, pl, _, _, _ = run_conv(backend, h, x, w, b, 1, p, 1, a, (oh, ow), what=f"bn {bn} {cell}")
        items = pl["m_tiles"] * pl["n_chunks"]
        print(f"BN {bn} {cell}: plan {pl}, oc {oc}, {n} x {oh}x{ow} pixels, {items} items on {sms} SMs, rel err {err:.2e}")
        assert (pl["bn"], pl["m_tiles"], pl["n_chunks"]) == (bn, m, -(-oc // bn))
        if cell == "kb1":
            assert pl["num_kb"] == 1
        else:
            assert pl["num_kb"] > pl["stages"] and pl["num_kb"] % pl["stages"], pl
        assert items > sms and sms % pl["n_chunks"], "a CTA's items must change n chunk"
        assert oc % bn, "ragged last n chunk"
        assert (oh * ow) % 128 and (n * oh * ow) % 128, "an M tile across two images and a part-empty last M tile"
    finally:
        lib().mnnb200_exec_destroy(h)


def probe_inputs(rng, probe, n, ic, oc, hw):
    """probe A: x = v + 2^-12 with v TF32-exact in [1, 2), w one-signed and TF32-exact: of the split terms only a_lo*w_hi carries
    the 2^-12.  Probe B is the mirror image, x TF32-exact and w = (u + 2^-12) 2^-6: only a_hi*w_lo carries it."""
    v = (1 + rng.integers(0, 1024, (n, ic) + hw) / 1024).astype(np.float32)
    u = (1 + rng.integers(0, 1024, (oc, ic, 1, 1)) / 1024).astype(np.float32)
    if probe == "A":
        x, w = v + np.float32(2.0 ** -12), u * np.float32(2.0 ** -6)
    else:
        x, w = v, (u + np.float32(2.0 ** -12)) * np.float32(2.0 ** -6)
    hi, lo = (x, w) if probe == "A" else (w, x)
    assert np.array_equal(tf32(hi), hi - np.float32(2.0 ** -12 * (1 if probe == "A" else 2.0 ** -6)))
    assert np.array_equal(tf32(lo), lo)
    b = rng.uniform(-0.05, 0.05, oc).astype(np.float32)
    return x, w, b


@pytest.mark.parametrize("bn", [32, 64, 128])
@pytest.mark.parametrize("probe", ["A", "B"])
def test_conv_f32_split_tf32_probe(backend, probe, bn):
    """a 1x1 layer with K = 64 whose inputs put the low part of x (A) or of w (B) into one split term alone: losing that term
    moves every output by more than twice its error bound, which the test checks in float64 before it runs the layer"""
    sms = sm_count()
    ic, oc = 64, {32: 24, 64: 56, 128: 200}[bn]
    m = next(m for m in range(1, 4 * sms) if plan_bn(oc, m, sms) == bn)
    n = 2
    hw = image_for_tiles(m, n)
    x, w, b = probe_inputs(np.random.default_rng(ord(probe) + bn), probe, n, ic, oc, hw)
    h = create_conv(backend, ic, oc, 1, 1, 0, 1, 0, w, b)
    try:
        oh, ow = resize(h, n, hw)
        ref, S = conv64(x, w, b, 1, 0, 1, 0)
        dropped = conv_ref(tf32(x), w, b, 1, 0, 1, 0) if probe == "A" else conv_ref(x, tf32(w), b, 1, 0, 1, 0)
        tol = conv_tolerance(S, b, 64)
        assert (np.abs(ref - dropped) > 2 * tol).all(), "the probe no longer separates the split term from the error bound"
        err, pl, _, _, y = run_conv(backend, h, x, w, b, 1, 0, 1, 0, (oh, ow), what=f"probe {probe}")
        assert (pl["bn"], pl["num_kb"]) == (bn, 2)
        plain = rel_err(conv_ref(tf32(x), tf32(w), b, 1, 0, 1, 0), ref)
        print(f"probe {probe} BN {bn}: split-TF32 rel err {err:.2e}, plain TF32 would give {plain:.2e}, "
              f"the lost term {rel_err(dropped, ref):.2e}; worst output at {float((np.abs(y - ref) / tol).max()):.2f} of its bound")
    finally:
        lib().mnnb200_exec_destroy(h)


def test_conv_f32_re_resize(backend):
    """one execution resized batch 1 (bn 32) -> a shape that plans bn 128 -> set_pad -> batch 1 again (bn 32): the weight tensor
    maps are remade at each change of width, and every output is checked"""
    sms = sm_count()
    ic, oc, a = 24, 200, 1
    rng = np.random.default_rng(200)
    _, w, b = conv_inputs(rng, ic, oc, 3, 1, 1)
    h = create_conv(backend, ic, oc, 3, 1, 1, 1, a, w, b)
    m128 = next(m for m in range(1, 4 * sms) if plan_bn(oc, m, sms) == 128)
    try:
        widths = []
        for n, hw, pad in ((1, (9, 11), (1, 1)), (2, image_for_tiles(m128), (1, 1)), (1, (10, 7), (0, 2))):
            if pad != (1, 1):
                assert lib().mnnb200_conv_f32_set_pad(h, *pad) == 0
            x = rng.standard_normal((n, ic) + hw).astype(np.float32)
            oh, ow = resize(h, n, hw)
            assert (oh, ow) == (natural_out(hw[0], 3, 1, pad[0], 1), natural_out(hw[1], 3, 1, pad[1], 1))
            err, pl, _, _, _ = run_conv(backend, h, x, w, b, 1, pad, 1, a, (oh, ow), what=f"resize to {n} x {hw}")
            print(f"re-resize {n} x {hw} pad {pad}: plan {pl}, rel err {err:.2e}")
            widths.append(pl["bn"])
        assert widths == [32, 128, 32]
    finally:
        lib().mnnb200_exec_destroy(h)


@functools.lru_cache(maxsize=None)
def mbv2_layers():
    """the 36 dense convs of MobileNet-v2 at batch 32 (the set tools/float_bench.py times), from the committed int8 graph: the
    architecture is the same, and only the geometry is taken"""
    from mnn_b200 import graph, mnn_file
    net = mnn_file.load(os.path.join(ROOT, "tests", "golden", "mbv2_int8.mnn"))
    shapes = graph.infer_shapes(net, (32, 3, 224, 224))
    out = []
    for op in graph.dense_convs(net):
        c = op.conv
        out.append((c.ic, c.oc, tuple(c.kernel), tuple(c.stride), tuple(op.attrs["resolved_pad"]), tuple(c.dilate),
                    tuple(op.attrs["in_shape"][2:]), tuple(shapes[op.outputs[0]][2:]), 2 if c.relu6 else int(c.relu)))
    assert len(out) == 36
    return out


MBV2_IMAGES = (0, 1, 31)            # image 31 holds the last M tiles


@pytest.mark.parametrize("layer", range(36))
def test_conv_f32_mobilenet_v2_layers(backend, layer):
    import torch
    ic, oc, k, s, p, d, ihw, ohw, a = mbv2_layers()[layer]
    n = 32
    rng = np.random.default_rng(1000 + layer)
    _, w, b = conv_inputs(rng, ic, oc, k, 1, 1)
    g = torch.Generator(device="cuda")
    g.manual_seed(layer)
    x = torch.randn((n, ic) + ihw, generator=g, device="cuda")
    h = create_conv(backend, ic, oc, k, s, p, d, a, w, b)
    try:
        assert lib().mnnb200_conv_f32_set_pad(h, *p) == 0
        assert resize(h, n, ihw, out=ohw) == ohw
        err, pl, _, _, _ = run_conv(backend, h, x, w, b, s, p, d, a, ohw, images=MBV2_IMAGES, what=f"layer {layer}")
        print(f"MobileNet-v2 layer {layer} ic {ic} oc {oc} k {k} s {s} {ihw}->{ohw}: plan {pl}, rel err {err:.2e}")
    finally:
        lib().mnnb200_exec_destroy(h)


def test_conv_f32_plan_query(backend):
    """NO_EXECUTION before resize, INVALID_VALUE for another kind of execution or no field array; count limits what is written,
    and reading the plan twice gives the same fields"""
    rng = np.random.default_rng(5)
    _, w, b = conv_inputs(rng, 8, 8, 3, 1, 1)
    _, wd, bd = conv_inputs(rng, 8, 8, 3, 1, 1, depthwise=True)
    h = create_conv(backend, 8, 8, 3, 1, 1, 1, 0, w, b)
    hd = create_conv(backend, 8, 8, 3, 1, 1, 1, 0, wd, bd, depthwise=True)
    try:
        f = (C.c_int * 7)(*([-7] * 7))
        assert lib().mnnb200_conv_f32_plan(h, f, 7) == NO_EXECUTION
        assert lib().mnnb200_conv_f32_plan(hd, f, 7) == INVALID_VALUE
        assert lib().mnnb200_conv_f32_plan(None, f, 7) == INVALID_VALUE
        resize(h, 1, 5)
        resize(hd, 1, 5, depthwise=True)
        assert lib().mnnb200_conv_f32_plan(hd, f, 7) == INVALID_VALUE
        assert lib().mnnb200_conv_f32_plan(h, None, 7) == INVALID_VALUE
        assert list(f) == [-7] * 7
        assert lib().mnnb200_conv_f32_plan(h, f, 3) == 0
        assert list(f) == [32, 1, 1, -7, -7, -7, -7]
        pl = plan(h)
        assert plan(h) == pl == dict(bn=32, n_chunks=1, m_tiles=1, num_kb=3, stages=pl["stages"], cp8=8, taps=9)
        assert pl["stages"] > 0
    finally:
        lib().mnnb200_exec_destroy(h)
        lib().mnnb200_exec_destroy(hd)


def test_conv_f32_resize_32bit_guards(backend):
    """resize returns NOT_SUPPORT one past each 32-bit indexing limit (M = n*oh*ow <= 2^31 - 129, n*ic*ih*iw and n*oc*oh*ow
    <= 2^31 - 1), each with the other two in range, accepts each limit itself, and a refused resize leaves the plan as it was.
    Only host arithmetic: nothing is allocated or launched."""
    rng = np.random.default_rng(6)
    _, w1, b1 = conv_inputs(rng, 1, 1, 1, 1, 1)
    _, w2, b2 = conv_inputs(rng, 1, 1024, 1, 1, 1)
    h1 = create_conv(backend, 1, 1, 1, 1, 0, 1, 0, w1, b1)
    h2 = create_conv(backend, 1, 1024, 1, 1, 0, 1, 0, w2, b2)

    def status(h, n, ih, iw, oh, ow):
        o, p = C.c_int(oh), C.c_int(ow)
        return lib().mnnb200_conv_f32_resize(h, n, ih, iw, C.byref(o), C.byref(p))

    try:
        lim = 2 ** 31 - 1
        assert status(h1, 1, 1, 1, lim - 128, 1) == 0                       # M = 2^31 - 129
        assert plan(h1)["m_tiles"] == -(-(lim - 128) // 128)
        before = plan(h1)
        assert status(h1, 1, 1, 1, (lim - 127) // 128, 128) == NOT_SUPPORT   # M = 2^31 - 128
        assert plan(h1) == before
        assert status(h1, 1, lim, 1, 1, 1) == 0                            # n*ic*ih*iw = 2^31 - 1
        before = plan(h1)
        assert status(h1, 2, 2 ** 30, 1, 1, 1) == NOT_SUPPORT               # 2^31
        assert plan(h1) == before
        assert status(h2, 1, 1, 1, 2 ** 21 - 1, 1) == 0                     # n*oc*oh*ow = 2^31 - 1024
        before = plan(h2)
        assert status(h2, 1, 1, 1, 2048, 1024) == NOT_SUPPORT               # 2^31
        assert plan(h2) == before
    finally:
        lib().mnnb200_exec_destroy(h1)
        lib().mnnb200_exec_destroy(h2)


def test_conv_f32_declines_grouped(backend):
    w = np.zeros((8, 4, 3, 3), np.float32)
    h = C.c_void_p()
    dd = desc(8, 8, 3, 1, 1, 1, 2, 0)
    assert lib().mnnb200_conv_f32_create(backend.runtime._h, C.byref(dd), w.ctypes.data_as(C.c_void_p), None, 0, C.byref(h)) == 2
    assert not h.value


def run_dw(backend, c, k, s, p, d, hw, n, a, seed):
    rng = np.random.default_rng(seed)
    x, w, b = conv_inputs(rng, c, c, k, hw, n, depthwise=True)
    h = create_conv(backend, c, c, k, s, p, d, a, w, b, depthwise=True)
    try:
        oh, ow = resize(h, n, hw, depthwise=True)
        (kh, kw), (sh, sw), (ph, pw), (dh, dw) = pair(k), pair(s), pair(p), pair(d)
        (ih, iw) = pair(hw)
        assert (oh, ow) == (natural_out(ih, kh, sh, ph, dh), natural_out(iw, kw, sw, pw, dw))
        y = execute(backend, h, x, (n, c, oh, ow), depthwise=True).cpu().numpy()
        ref, S = conv64(x, w, b, s, p, d, a, groups=c)
        check_elements(y, ref, dw_tolerance(S, b, kh * kw), "depthwise")
        assert rel_err(y, ref) <= 1e-5
    finally:
        lib().mnnb200_exec_destroy(h)


@pytest.mark.parametrize("case", [(32, 3, 1, 1, 1, 112, 1, 2), (144, 3, 2, 1, 1, 56, 2, 2), (960, 3, 1, 1, 1, 7, 32, 1),
                                  (64, 5, 1, 4, 2, 14, 2, 0), (24, 3, 2, 0, 1, 15, 3, 1)],
                         ids=lambda c: "c%d_k%d_s%d_p%d_d%d_hw%d_n%d_a%d" % c)
def test_dwconv_f32_matches_float64(backend, case):
    c, k, s, p, d, hw, n, a = case
    run_dw(backend, c, k, s, p, d, hw, n, a, c + k * 7 + hw)


# name: channels, kernel, stride, pad, dilation, (ih, iw), batch, act
DW_GEOMETRY = {
    "k3x5_s1x2_p2x2_d2x1": (24, (3, 5), (1, 2), (2, 2), (2, 1), (13, 17), 2, 1),
    "k5x3_s2x1_p1x3_d1x2": (20, (5, 3), (2, 1), (1, 3), (1, 2), (16, 11), 2, 0),
    "k3_p1x0_ih9_iw14": (7, 3, 1, (1, 0), 1, (9, 14), 3, 2),
}


@pytest.mark.parametrize("name", list(DW_GEOMETRY))
def test_dwconv_f32_geometry(backend, name):
    run_dw(backend, *DW_GEOMETRY[name], seed=sum(map(ord, name)))


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
